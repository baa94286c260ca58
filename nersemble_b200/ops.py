"""Tensor-level wrappers over the libnsb C ABI (include/nsb.h).

PyTorch is used for device memory and streams only; all arithmetic of the hot path runs in
the hand-written sm_90a kernels.  There is no CPU fallback: non-CUDA tensors raise.
"""
from __future__ import annotations

import ctypes as C
import functools
from dataclasses import dataclass
from typing import Dict, Optional, Sequence

import torch

from . import _lib, packing

_F32 = torch.float32

# Deformation MLP of the inference kernels on wgmma (the "tcgen05" flag keeps its original name; NativeParams.build(tcgen05=...)
# overrides it per instance;
# NSB_TCGEN05=0/1 in the environment overrides the default).
import os as _os
USE_TCGEN05 = _os.environ.get("NSB_TCGEN05", "1") == "1"


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _need_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("nersemble_b200 ops need CUDA tensors (there is no CPU fallback)")


_WORKSPACES: dict = {}


def _workspace(name: str, nbytes: int, dev) -> torch.Tensor:
    """Reusable scratch buffers, one per (name, device, STREAM): contents are undefined between calls and ops on one
    stream are ordered, so two streams (trainer + viewer thread, engine/nersemble_trainer.py:38-40) never share one."""
    key = (name, str(dev), torch.cuda.current_stream(dev).cuda_stream)
    t = _WORKSPACES.get(key)
    if t is None or t.numel() < nbytes:
        t = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        _WORKSPACES[key] = t
    return t


_ROW_QUANTUM = 1 << 16


def _rows(n: int, tail=(), dtype=_F32, device=None, zero: bool = False) -> torch.Tensor:
    """[n, *tail] as a view of an allocation rounded up to 65 536 rows.  The packed sample count changes every training
    step (stratified jitter); exact-size allocations of the large per-sample buffers (2.7 GB of saved activations at
    1.8 M samples) then miss the caching allocator's free blocks whenever the count grows and fall through to
    cudaMalloc, which costs host time on every forward and more with the backward buffers."""
    n_alloc = max(((int(n) + _ROW_QUANTUM - 1) // _ROW_QUANTUM) * _ROW_QUANTUM, 1)
    t = (torch.zeros if zero else torch.empty)((n_alloc,) + tuple(tail), dtype=dtype, device=device)
    return t[:n]


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _f32c(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    if t is None:
        return None
    return t.detach().to(_F32).contiguous()


@dataclass
class NativeParams:
    """Device-resident parameters in the kernels' layouts (see packing.py)."""
    tables: Optional[torch.Tensor]          # half [entries, 32, 2]
    deform_bias: Optional[torch.Tensor]     # float [776]
    field_packed: Optional[torch.Tensor]    # half, fragment order
    warp_codes: Optional[torch.Tensor]      # half [T, 128]
    blend_codes: Optional[torch.Tensor]     # float [T, 32]
    aabb: torch.Tensor            # float [2,3] (cpu copy kept in aabb_list)
    levels: dict
    n_timesteps: int
    field_packed_t: Optional[torch.Tensor] = None     # half, transposed field weights (backward)
    deform_packed_t: Optional[torch.Tensor] = None    # half, transposed deformation weights (backward)
    deform_packed_tb: Optional[torch.Tensor] = None   # half, fragment order, no warp-code columns
    deform_code_w: Optional[list] = None              # (stem_w[0], stem_w[4], stem_b[0], stem_b[4]): per-sample code bias
    deform_code_bias: Optional[torch.Tensor] = None   # float [T, 2, 128]
    deform_packed_umma: Optional[torch.Tensor] = None # half, wgmma core-matrix order (inference kernels; opt-in)
    deform_packed_pe_t: Optional[torch.Tensor] = None # half, transposed posenc columns of layers 0 / 4 (deform_input_grad)

    def __post_init__(self):
        self.aabb_list = [float(v) for v in self.aabb.detach().cpu().reshape(-1)]
        lv = self.levels
        for l in range(lv["n_levels"]):
            if lv["hashed"][l]:
                e = lv["entries"][l]
                assert e & (e - 1) == 0, "hashed levels must have power-of-two size"
        if self.tables is not None:
            assert self.tables.dtype == torch.float16 and self.tables.shape[1:] == (32, 2)
            assert self.tables.shape[0] == lv["total_entries"]

    @staticmethod
    def build(*, tables, time_emb, aabb, levels, base_w=None, head_w=None, deform=None, time_emb_deform=None,
              device="cuda", tcgen05: Optional[bool] = None) -> "NativeParams":
        """tables: [entries,32,2] (any float dtype); base_w/head_w: lists of [out,in] matrices;
        deform: dict(stem_w, stem_b, r_w, r_b, v_w, v_b) or None."""
        dev = torch.device(device)
        if time_emb is not None and base_w is not None and time_emb.shape[-1] != 32:
            raise ValueError(f"time_emb must be [T, 32] (one blend weight per ensemble member), got {tuple(time_emb.shape)}")
        if deform is not None and (time_emb_deform is None or time_emb_deform.shape[-1] != 128):
            raise ValueError("time_emb_deform must be [T, 128] (SE3DeformationFieldConfig.warp_code_dim = 128)")
        tab = None if tables is None else tables.detach().to(dev).half().contiguous()
        fp = fpt = None
        db = wc = dtb = dpt = dcb = None
        if deform is not None:
            sw, sb = [w.to(dev) for w in deform["stem_w"]], [b.to(dev) for b in deform["stem_b"]]
        if base_w is not None and deform is not None:      # the training path: one gather for all five buffers
            dtb, dpt, fp, fpt = packing.pack_all_fast(sw, deform["r_w"].to(dev), deform["v_w"].to(dev),
                                                          [w.detach().to(dev) for w in base_w], [w.detach().to(dev) for w in head_w])
        elif base_w is not None:
            fp, fpt = packing.pack_field_fast([w.detach().to(dev) for w in base_w], [w.detach().to(dev) for w in head_w])
        elif deform is not None:
            dtb, dpt = packing.pack_deform_weights_fast(sw, deform["r_w"].to(dev), deform["v_w"].to(dev))
        if deform is not None:
            db = packing.deform_bias_vector(sb, deform["r_b"].to(dev), deform["v_b"].to(dev))
            wc = time_emb_deform.detach().to(dev).half().contiguous()
            dcb = packing.deform_code_bias(sw, sb, wc)
        te = None if time_emb is None else time_emb.detach().to(dev).float().contiguous()
        n_t = int(time_emb.shape[0]) if time_emb is not None else (int(time_emb_deform.shape[0]) if time_emb_deform is not None else 1)
        P = NativeParams(tab, db, fp, wc, te, aabb.detach().float().cpu(), levels, n_t)
        if deform is not None:
            P.deform_packed_tb, P.deform_code_bias, P.deform_packed_t = dtb, dcb, dpt
            P.deform_code_w = [sw[0].detach(), sw[4].detach(), sb[0].detach(), sb[4].detach()]
            if USE_TCGEN05 if tcgen05 is None else tcgen05:     # packed lazily, by the first inference call (c_params)
                P._umma_src = (sw, deform["r_w"].to(dev), deform["v_w"].to(dev))
        P.field_packed_t = fpt
        return P

    def frame_table(self, uniform_time: float, window_hash, disable_initial: bool, soft_transition: bool) -> Optional[torch.Tensor]:
        """float [total_entries, 2]: the tables blended with the member weights of ONE timestep (nsb_blend_tables), for
        calls whose samples all carry `uniform_time` (a camera frame).  Cached per (timestep, window, table version); None
        when the wgmma inference kernels (the only ones that read it) are not in use."""
        if getattr(self, "_umma_src", None) is None or self.tables is None or self.blend_codes is None:
            return None
        import numpy as np
        tsi = int(np.rint(np.float32(uniform_time) * np.float32(self.n_timesteps - 1)))     # the kernels' __float2int_rn(t * (T - 1))
        tsi = min(max(tsi, 0), self.n_timesteps - 1)
        key = (tsi, None if window_hash is None else float(window_hash), bool(disable_initial), bool(soft_transition),
               self.tables.data_ptr(), self.tables._version, self.blend_codes.data_ptr(), self.blend_codes._version)
        cached = getattr(self, "_frame", None)
        if cached is None or cached[0] != key:
            out = cached[1] if cached is not None else torch.empty((self.tables.shape[0], 2), dtype=_F32, device=self.tables.device)
            opts = make_opts(window_hash, None, True, True, disable_initial, soft_transition)
            cp = self.c_params()
            _lib.check(_lib.load().nsb_blend_tables(C.byref(cp), C.byref(opts), tsi, 1, int(self.tables.shape[0]), _ptr(out), _stream()),
                       "nsb_blend_tables")
            self._frame = cached = (key, out)
        return cached[1]

    def timestep_tables(self, window_hash, disable_initial: bool, soft_transition: bool) -> Optional[torch.Tensor]:
        """float [T, total_entries, 2]: frame_table of every timestep, stacked (one nsb_blend_tables pass), for calls whose
        samples carry mixed timesteps: the gather then reads one 8 B entry per corner instead of a 128 B line.  Cached
        per (window, table version).  None when the wgmma inference kernels are not in use, or when the stack would be
        more than twice the size of the line tables (T > 32): the line gather is then the cheaper path."""
        if getattr(self, "_umma_src", None) is None or self.tables is None or self.blend_codes is None:
            return None
        T, E = self.n_timesteps, int(self.tables.shape[0])
        if T * E * 8 > 2 * self.tables.nbytes or T * E > 0xFFFFFFFF:      # the kernels index the stack in 32 bits
            return None
        key = (None if window_hash is None else float(window_hash), bool(disable_initial), bool(soft_transition),
               self.tables.data_ptr(), self.tables._version, self.blend_codes.data_ptr(), self.blend_codes._version)
        cached = getattr(self, "_stack", None)
        if cached is None or cached[0] != key:
            out = cached[1] if cached is not None else torch.empty((T, E, 2), dtype=_F32, device=self.tables.device)
            opts = make_opts(window_hash, None, True, True, disable_initial, soft_transition)
            cp = self.c_params()
            _lib.check(_lib.load().nsb_blend_tables(C.byref(cp), C.byref(opts), 0, T, E, _ptr(out), _stream()), "nsb_blend_tables")
            self._stack = cached = (key, out)
        return cached[1]

    def at_time(self, t: float) -> "NativeParams":
        """A one-timestep view of the parameters at the continuous time t (DESIGN 4.2g): the tables and every weight are
        shared with self; blend_codes [1,32] and deform_code_bias [1,2,128] are the time_lerp of the rows floor(u) and
        floor(u) + 1, warp_codes [1,128] the fp16 of the interpolated fp32 codes (only the training backward reads it).
        With T = 1 every kernel maps every sample to row 0, so any render, field or mesh call on the view answers at t.
        At a snapped integer time the rows are the parent's row bit for bit.  Built on the device without a host
        synchronisation; cached per (rows, lam, parameter versions)."""
        i0, i1, lam = time_lerp(t, self.n_timesteps)
        vers = tuple((x.data_ptr(), x._version) if x is not None else None
                     for x in (self.blend_codes, self.deform_code_bias, self.warp_codes))
        key = (i0, lam, vers)
        cached = getattr(self, "_at_time", None)
        if cached is None or cached[0] != key:
            def rows(x):
                if x is None:
                    return None
                a = x[i0:i0 + 1]
                if lam == 0.0:
                    return a.clone()
                return _lerp_f32(a.float(), x[i1:i1 + 1].float(), lam).to(x.dtype)
            if self.deform_packed_umma is None and getattr(self, "_umma_src", None) is not None:
                self.deform_packed_umma = packing.pack_deform_umma_fast(*self._umma_src)     # shared, packed once
            V = NativeParams(self.tables, self.deform_bias, self.field_packed, rows(self.warp_codes), rows(self.blend_codes),
                             self.aabb, self.levels, 1)
            V.field_packed_t, V.deform_packed_t, V.deform_packed_tb = self.field_packed_t, self.deform_packed_t, self.deform_packed_tb
            V.deform_code_w, V.deform_code_bias = self.deform_code_w, rows(self.deform_code_bias)
            V.deform_packed_umma, V.deform_packed_pe_t = self.deform_packed_umma, self.deform_packed_pe_t
            if getattr(self, "_umma_src", None) is not None:
                V._umma_src = self._umma_src
            self._at_time = cached = (key, V)
        V = cached[1]
        V.tables = self.tables          # the plugin swaps in its current tables before every call
        return V

    def pe_t(self) -> torch.Tensor:
        """packing.pack_deform_pe_t of the stem weights, packed on first use (only the deformation input gradient reads it)."""
        if self.deform_packed_pe_t is None:
            if self.deform_code_w is None:
                raise RuntimeError("the deformation input gradient needs deformation weights (NativeParams.build(deform=...))")
            self.deform_packed_pe_t = packing.pack_deform_pe_t(self.deform_code_w[0], self.deform_code_w[1])
        return self.deform_packed_pe_t

    def c_params(self, inference: bool = False, frame: Optional[torch.Tensor] = None) -> _lib.FieldParams:
        """inference: the call saves nothing for a backward pass -- the kernels may then run the deformation MLP on
        wgmma, which takes its weights in another order (packed here on first use: a training step never pays).
        frame: a frame_table [E, 2] (every sample has its timestep) or a timestep_tables stack [T, E, 2]."""
        if inference and self.deform_packed_umma is None and getattr(self, "_umma_src", None) is not None:
            self.deform_packed_umma = packing.pack_deform_umma_fast(*self._umma_src)
        p = getattr(self, "_cp", None)      # the level table / aabb part never changes: fill it once (host time matters:
        fresh = p is None                   # a training step has little GPU time to hide host work behind)
        if fresh:
            p = self._cp = _lib.FieldParams()
        p.tables = _ptr(self.tables)
        p.deform_bias = _ptr(self.deform_bias)
        p.deform_packed_tb = _ptr(self.deform_packed_tb)
        p.deform_code_bias = _ptr(self.deform_code_bias)
        p.deform_packed_umma = _ptr(self.deform_packed_umma) if inference else None
        p.frame_table = _ptr(frame) if (inference and self.deform_packed_umma is not None) else None
        p.frame_stride = int(frame.shape[1]) if (p.frame_table and frame.dim() == 3) else 0
        p.field_packed = _ptr(self.field_packed)
        p.warp_codes = _ptr(self.warp_codes)
        p.blend_codes = _ptr(self.blend_codes)
        p.n_timesteps = self.n_timesteps
        if fresh:
            for i, v in enumerate(self.aabb_list):
                p.aabb[i] = v
            lv = self.levels
            p.levels.n_levels = lv["n_levels"]
            for l in range(lv["n_levels"]):
                p.levels.scale[l] = lv["scale"][l]
                p.levels.res[l] = lv["res"][l]
                p.levels.entries[l] = lv["entries"][l]
                p.levels.offset[l] = lv["offset"][l]
                p.levels.hashed[l] = lv["hashed"][l]
        return p


# Continuous time (DESIGN 4.2g).  "nearest" rounds a time to the nearest captured timestep, as the reference does;
# "linear" interpolates the per-timestep codes between the two neighbouring timesteps.
TIME_INTERPOLATIONS = ("nearest", "linear")
TIME_SNAP = 2.0 ** -10      # timesteps: fp32 times k / (T - 1) land a few ulp off k (2.4e-4 timesteps at T = 2000)


def time_lerp(t: float, n_timesteps: int):
    """(i0, i1, lam) of time t over n_timesteps timesteps, in fp32 as the kernels form it (nsb_common.cuh
    sample_time_u): u = clamp(t * (T - 1), 0, T - 1), snapped to rint(u) when within TIME_SNAP of it; i0 = floor(u),
    i1 = min(i0 + 1, T - 1), lam = u - i0.  A per-timestep quantity q at t is fmaf(lam, q[i1] - q[i0], q[i0])."""
    import numpy as np
    T = int(n_timesteps)
    if T < 1:
        raise ValueError(f"time_lerp: n_timesteps must be >= 1, got {n_timesteps!r}")
    tm = np.float32(T - 1)
    with np.errstate(invalid="ignore", over="ignore"):
        u = np.float32(np.float32(t) * tm)
    u = np.float32(min(max(np.fmax(u, np.float32(0.0)), np.float32(0.0)), tm))     # fmaxf: NaN -> 0
    r = np.float32(np.rint(u))
    if abs(np.float32(u - r)) <= np.float32(TIME_SNAP):
        u = r
    i0 = min(int(np.floor(u)), T - 1)
    return i0, min(i0 + 1, T - 1), float(np.float32(u - np.float32(i0)))


def _lerp_f32(a: torch.Tensor, b: torch.Tensor, lam) -> torch.Tensor:
    """fmaf(lam, b - a, a) in fp32 (lam a float or a tensor broadcasting against a): b - a rounded to fp32, then one
    product and sum in fp64 (exact for the 24-bit lam times the 24-bit difference) and one rounding to fp32."""
    lam = lam.double() if torch.is_tensor(lam) else float(lam)
    return (a.double() + (b - a).double() * lam).float()


def time_lerp_rows(times: torch.Tensor, n_timesteps: int):
    """time_lerp of every time of a tensor, on its device: (i0 [n] int64, i1 [n] int64, lam [n] fp32)."""
    T = int(n_timesteps)
    t = times.detach().reshape(-1).to(_F32)
    tm = float(T - 1)
    u = torch.nan_to_num(t * tm, nan=0.0).clamp(0.0, tm)
    r = torch.round(u)
    u = torch.where((u - r).abs() <= TIME_SNAP, r, u)
    i0 = u.floor().long().clamp(max=T - 1)
    return i0, (i0 + 1).clamp(max=T - 1), u - i0.to(_F32)


def time_codes(P: NativeParams, times: torch.Tensor) -> Dict[str, torch.Tensor]:
    """Per-time interpolated codes for the per-sample-code kernels (field_forward(sample_blend_codes=,
    sample_warp_codes=)), on the device without a host synchronisation: times [n] -> {"blend_codes" [n,32] fp32,
    "warp_codes" [n,128] fp32 (with a deformation field)}, each time_lerp of the parameters' rows."""
    i0, i1, lam = time_lerp_rows(times, P.n_timesteps)
    lam = lam[:, None]
    out = {}
    if P.blend_codes is not None:
        out["blend_codes"] = _lerp_f32(P.blend_codes[i0], P.blend_codes[i1], lam)
    if P.warp_codes is not None:
        wc = P.warp_codes.float()
        out["warp_codes"] = _lerp_f32(wc[i0], wc[i1], lam)
    return out


def _check_time_interpolation(time_interpolation, who: str) -> bool:
    """True for "linear"; ValueError for anything not in TIME_INTERPOLATIONS."""
    if time_interpolation not in TIME_INTERPOLATIONS:
        raise ValueError(f"{who}: time_interpolation must be one of {TIME_INTERPOLATIONS}, got {time_interpolation!r}")
    return time_interpolation == "linear"


def make_opts(window_hash: Optional[float], window_deform: Optional[float], use_deformation: bool,
              compute_rgb: bool, disable_initial: bool = True, soft_transition: bool = True) -> _lib.FieldOpts:
    """nsb_field_opts for the given schedule values (memoised: the windows change once per training step at most, and
    the struct is only read)."""
    return _make_opts(None if window_hash is None else float(window_hash), None if window_deform is None else float(window_deform),
                      bool(use_deformation), bool(compute_rgb), bool(disable_initial), bool(soft_transition))


@functools.lru_cache(maxsize=64)
def _make_opts(window_hash, window_deform, use_deformation, compute_rgb, disable_initial, soft_transition) -> _lib.FieldOpts:
    o = _lib.FieldOpts()
    sc, bi = packing.blend_fold(window_hash, 32, disable_initial, soft_transition)
    for h in range(32):
        o.cw_scale[h] = sc[h]
        o.cw_bias[h] = bi[h]
    for j, w in enumerate(packing.deform_window(window_deform)):
        o.pe_window[j] = w
    o.use_deformation = int(use_deformation)
    o.compute_rgb = int(compute_rgb)
    return o


def field_forward(P: NativeParams, *, window_hash=None, window_deform=None, use_deformation=True,
                  origins=None, directions=None, ray_times=None, t_starts=None, t_ends=None, ray_indices=None,
                  positions=None, sample_times=None, sample_directions=None, sample_blend_codes=None,
                  sample_warp_codes=None, n_samples_dev: Optional[torch.Tensor] = None,
                  given_feat: Optional[torch.Tensor] = None, uniform_time: Optional[float] = None,
                  want: Sequence[str] = ("sigma", "rgb", "offsets"),
                  disable_initial: bool = True, soft_transition: bool = True, line_gather: bool = False) -> Dict[str, torch.Tensor]:
    """Fused deformation + hash ensemble + field MLPs for packed samples (nsb_field_forward).
    Inference calls gather member-blended tables (NativeParams.frame_table for a uniform_time, timestep_tables
    otherwise) when the wgmma kernels run; line_gather=True forces the per-sample blend of the 128 B table lines."""
    lib = _lib.load()
    keep = []
    s = _lib.Samples()
    n = _fill_samples(s, keep, origins=origins, directions=directions, ray_times=ray_times, t_starts=t_starts, t_ends=t_ends,
                      ray_indices=ray_indices, positions=positions, sample_times=sample_times,
                      sample_directions=sample_directions, sample_blend_codes=sample_blend_codes)
    dev = (origins if origins is not None else positions).device
    if sample_blend_codes is not None:
        assert tuple(sample_blend_codes.shape) == (n, 32)
    if sample_warp_codes is not None:
        _fill_sample_code_bias(P, s, keep, sample_warp_codes, n, dev)
    if n_samples_dev is not None:      # the arrays hold `n` slots, the device scalar says how many are samples (no host sync)
        assert n_samples_dev.dtype == torch.int64 and n_samples_dev.is_cuda and n_samples_dev.numel() == 1
        s.n_samples_dev = _ptr(n_samples_dev); keep.append(n_samples_dev)
    if given_feat is not None:         # pre-pass reuse: the blended features are an INPUT, the table gather is skipped
        assert given_feat.dtype == torch.float16 and given_feat.is_contiguous() and tuple(given_feat.shape) == (n, 32)
        assert "feat" not in want and "corner_vals" not in want, "given_feat: feat / corner_vals come from the pre-pass"
        _need_cuda(given_feat)
        s.given_feat = _ptr(given_feat); keep.append(given_feat)
    out = {}
    o = _lib.FieldOut()
    if "sigma" in want:
        out["sigma"] = _rows(n, (), _F32, dev); o.sigma = _ptr(out["sigma"])
    if "rgb" in want:
        out["rgb"] = _rows(n, (3,), _F32, dev); o.rgb = _ptr(out["rgb"])
    if "offsets" in want:
        if use_deformation:
            out["offsets"] = _rows(n, (3,), _F32, dev); o.offsets = _ptr(out["offsets"])
        else:
            out["offsets"] = _rows(n, (3,), _F32, dev, zero=True)
    if "feat" in want:
        out["feat"] = _rows(n, (32,), torch.float16, dev); o.feat = _ptr(out["feat"])
    if "xs" in want:
        out["xs"] = _rows(n, (4,), _F32, dev); o.xs = _ptr(out["xs"])
    if "corner_vals" in want:   # training forward: blended corner values, so the backward does not re-gather the tables
        out["corner_vals"] = _rows(n, (16, 8, 2), torch.float16, dev)
        o.corner_vals = _ptr(out["corner_vals"])
    if "deform_acts" in want:   # training forward: stem activations + posenc fragments for nsb_deform_backward
        n_tiles = (n + 127) // 128
        out["deform_acts"] = _rows(n_tiles * 128, (384,), torch.int32, dev).view(n_tiles, 8, 6, 8, 32, 4)
        out["deform_enc"] = _rows(n_tiles * 128, (24,), torch.int32, dev).view(n_tiles, 8, 3, 32, 4)
        o.deform_acts, o.deform_enc = _ptr(out["deform_acts"]), _ptr(out["deform_enc"])
    if n == 0:
        return out
    opts = make_opts(window_hash, window_deform, use_deformation, "rgb" in want, disable_initial, soft_transition)
    inference = (use_deformation and n_samples_dev is None and given_feat is None and sample_warp_codes is None
                 and not any(k in want for k in ("feat", "xs", "corner_vals", "deform_acts")))
    frame = None
    if inference and ("sigma" in want or "rgb" in want):
        frame = _blended_tables(P, uniform_time, window_hash, disable_initial, soft_transition, line_gather, sample_blend_codes)
    cp = P.c_params(inference=inference, frame=frame)
    rc = lib.nsb_field_forward(C.byref(cp), C.byref(opts), C.byref(s), C.byref(o), _stream())
    _lib.check(rc, "nsb_field_forward")
    return out


def _fill_sample_code_bias(P: NativeParams, s, keep, sample_warp_codes, n: int, dev) -> None:
    """Component API (explicit per-sample warp codes): the kernels take the code columns of layers 0 / 4 as a per-sample
    bias, W_code . code + b (fp16-rounded operands, fp32 accumulate)."""
    assert sample_warp_codes.shape == (n, 128) and P.deform_code_w is not None
    if n > (1 << 24):
        raise RuntimeError("per-sample warp codes: at most 2^24 samples per call")
    w0, w4, b0, b4 = P.deform_code_w
    scb = packing.deform_code_bias({0: w0, 4: w4}, {0: b0, 4: b4}, sample_warp_codes.to(dev))
    s.sample_code_bias = _ptr(scb); keep.append(scb)


# Scale of the fp16 deltas of the deformation input gradient.  Its cotangents are unit normals over the box extent or
# caller vectors of similar size, and the chain only shrinks them (head weights << 1): 1024 keeps the deltas in fp16's
# normal range without coming near its maximum.
VJP_LOSS_SCALE = 1024.0
NORMAL_SPACES = ("canonical", "observation")


def deform_input_grad(P: NativeParams, u: torch.Tensor, *, window_deform=None, loss_scale: float = VJP_LOSS_SCALE,
                      sample_warp_codes: Optional[torch.Tensor] = None, n_samples_dev: Optional[torch.Tensor] = None,
                      out: Optional[torch.Tensor] = None, **sample_kw) -> torch.Tensor:
    """J^T u [n,3] of the SE(3) deformation with respect to its NORMALISED input position (nsb_deform_input_grad):
    offset(p_n) = field_forward(...)["offsets"], J = d offset / d p_n through the windowed positional encoding, the stem,
    both heads, the exponential map and the direct term (R - I) p_n.  u [n,3]: cotangent of the normalised offsets.
    Samples as in field_forward (positions / sample_times, or origins / directions / t_starts / t_ends / ray_indices /
    ray_times), with table warp codes or sample_warp_codes [n,128].  Written into `out` (float32 [n,3], contiguous) when
    given; rows beyond *n_samples_dev are not touched.
    Nothing a forward saved is needed; not differentiable."""
    keep: list = []
    s = _lib.Samples()
    n = _fill_samples(s, keep, **sample_kw)
    u = _f32c(u).reshape(-1, 3)
    _need_cuda(u)
    assert u.shape[0] == n, (u.shape, n)
    dev = u.device
    if sample_warp_codes is not None:
        _fill_sample_code_bias(P, s, keep, sample_warp_codes, n, dev)
    if n_samples_dev is not None:
        assert n_samples_dev.dtype == torch.int64 and n_samples_dev.is_cuda and n_samples_dev.numel() == 1
        s.n_samples_dev = _ptr(n_samples_dev); keep.append(n_samples_dev)
    if out is None:
        out = _rows(n, (3,), _F32, dev)
    assert out.dtype == _F32 and out.is_cuda and out.is_contiguous() and tuple(out.shape) == (n, 3)
    if n == 0:
        return out
    a = _lib.DeformVjpArgs()
    a.deform_packed_t, a.deform_packed_pe_t = _ptr(P.deform_packed_t), _ptr(P.pe_t())
    a.u, a.loss_scale, a.d_pn = _ptr(u), float(loss_scale), _ptr(out)
    opts = make_opts(None, window_deform, True, False)
    cp = P.c_params()
    _lib.check(_lib.load().nsb_deform_input_grad(C.byref(cp), C.byref(opts), C.byref(s), C.byref(a), _stream()),
               "nsb_deform_input_grad")
    return out


# Scale of the fp16 tangent rows of the deformation Jacobian (nsb_deform_jacobian / nsb_deform_inverse).  The largest
# posenc tangent is window * 2 pi 2^6 = 402 per unit of p_n; scaled by 1/16 it is 25, so the stem's tangent rows stay three
# orders of magnitude below fp16's maximum (65504) while the entries that matter stay far above its smallest normal (6.1e-5).
JVP_TANGENT_SCALE = 1.0 / 16.0
INVERSE_MAX_ITER = 64
# Render weight below which a sample takes no part in render_flow (DESIGN 4.2f): such samples are nearly transparent space,
# and inverting the warp for them is most of the cost of a flow pass for almost none of its weight.
# accumulation - flow_weight reports, per ray, the weight this leaves out.
FLOW_MIN_WEIGHT = 1e-3


def _positions_samples(sample_kw, who: str):
    if any(sample_kw.get(k) is not None for k in ("origins", "directions", "t_starts", "t_ends", "ray_indices", "ray_times")):
        raise ValueError(f"{who}: positions-based samples only (positions, sample_times)")
    if sample_kw.get("positions") is None:
        raise ValueError(f"{who}: positions are required")


def deform_jacobian(P: NativeParams, *, window_deform=None, sample_warp_codes: Optional[torch.Tensor] = None,
                    n_samples_dev: Optional[torch.Tensor] = None, **sample_kw) -> Dict[str, torch.Tensor]:
    """Offsets and Jacobian of the SE(3) deformation at given points (nsb_deform_jacobian), in one forward-mode pass:
    {"offsets" [n,3]: the normalised offsets field_forward(want=("offsets",)) reports (equal up to fp16 operand rounding),
     "jacobian" [n,3,3]: J[i][k] = d offset_i / d p_n[k], p_n the normalised position -- the J whose transpose
     deform_input_grad applies}.  Samples: positions [n,3] with sample_times [n] (table warp codes of the rounded
    timestep) or sample_warp_codes [n,128].  Not differentiable."""
    _positions_samples(sample_kw, "deform_jacobian")
    keep: list = []
    s = _lib.Samples()
    n = _fill_samples(s, keep, **sample_kw)
    dev = sample_kw["positions"].device
    if sample_warp_codes is not None:
        _fill_sample_code_bias(P, s, keep, sample_warp_codes, n, dev)
    if n_samples_dev is not None:
        assert n_samples_dev.dtype == torch.int64 and n_samples_dev.is_cuda and n_samples_dev.numel() == 1
        s.n_samples_dev = _ptr(n_samples_dev); keep.append(n_samples_dev)
    out = {"offsets": torch.empty((n, 3), dtype=_F32, device=dev), "jacobian": torch.empty((n, 3, 3), dtype=_F32, device=dev)}
    if n == 0:
        return out
    a = _lib.DeformJacArgs()
    a.tangent_scale, a.offsets, a.jacobian = JVP_TANGENT_SCALE, _ptr(out["offsets"]), _ptr(out["jacobian"])
    opts = make_opts(None, window_deform, True, False)
    cp = P.c_params()
    _lib.check(_lib.load().nsb_deform_jacobian(C.byref(cp), C.byref(opts), C.byref(s), C.byref(a), _stream()),
               "nsb_deform_jacobian")
    return out


def _check_newton(max_iter, tol, who: str):
    import math
    if not isinstance(max_iter, int) or not 1 <= max_iter <= INVERSE_MAX_ITER:
        raise ValueError(f"{who}: max_iter must be an int in 1..{INVERSE_MAX_ITER}, got {max_iter!r}")
    if not (math.isfinite(float(tol)) and float(tol) > 0):
        raise ValueError(f"{who}: tol must be finite and > 0, got {tol!r}")


def deform_inverse(P: NativeParams, targets: torch.Tensor, *, sample_times: Optional[torch.Tensor] = None,
                   uniform_time: Optional[float] = None, init: Optional[torch.Tensor] = None, window_deform=None,
                   sample_warp_codes: Optional[torch.Tensor] = None, max_iter: int = 20, tol: float = 1e-4,
                   n_samples_dev: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """Inverse of the deformation (nsb_deform_inverse): for each target c [n,3] -- a world position of the warped hash
    input, i.e. an observed position plus its normalised offset, as the field kernels form it -- the observed position p
    whose warp at the given time lands on c: the root of p_n + D^-1 offset(p_n) - c_n by damped Newton in the kernel.
    Time per point (sample_times [n]) or for all (uniform_time), or per-point warp codes (sample_warp_codes [n,128]).
    init [n,3]: initial guesses (default: the targets).  tol: on |F|inf in normalised units (1e-4 is about 1/20 of a voxel
    of a 512^3 grid).  Returns {"positions" [n,3] world (the best trial; the initial guess bit for bit when it already
    converged), "residual" [n] (|F|inf there), "iterations" [n] int32, "converged" [n] bool, "status" [n] int32
    (_lib.INV_CONVERGED / INV_NOT_CONVERGED / INV_SINGULAR)}.  n_samples_dev: optional device int64 scalar, the number of
    leading points to solve (the rest of every output is left as it was allocated).  Not differentiable."""
    _check_newton(max_iter, tol, "deform_inverse")
    if (sample_times is not None) + (uniform_time is not None) + (sample_warp_codes is not None) > 1:
        raise ValueError("deform_inverse: give one of sample_times, uniform_time, sample_warp_codes")
    targets = _f32c(targets).reshape(-1, 3)
    _need_cuda(targets)
    n, dev = int(targets.shape[0]), targets.device
    if uniform_time is not None:
        sample_times = torch.full((n,), float(uniform_time), dtype=_F32, device=dev)
    keep: list = []
    s = _lib.Samples()
    _fill_samples(s, keep, positions=targets, sample_times=sample_times)
    if sample_warp_codes is not None:
        _fill_sample_code_bias(P, s, keep, sample_warp_codes, n, dev)
    if n_samples_dev is not None:
        assert n_samples_dev.dtype == torch.int64 and n_samples_dev.is_cuda and n_samples_dev.numel() == 1
        s.n_samples_dev = _ptr(n_samples_dev); keep.append(n_samples_dev)
    a = _lib.DeformInvArgs()
    if init is not None:
        init = _f32c(init).reshape(-1, 3)
        _need_cuda(init)
        assert init.shape[0] == n, (init.shape, n)
        a.init = _ptr(init); keep.append(init)
    out = {"positions": torch.empty((n, 3), dtype=_F32, device=dev), "residual": torch.empty((n,), dtype=_F32, device=dev),
           "iterations": torch.empty((n,), dtype=torch.int32, device=dev), "status": torch.empty((n,), dtype=torch.int32, device=dev)}
    if n > 0:
        a.tangent_scale, a.max_iter, a.tol = JVP_TANGENT_SCALE, int(max_iter), float(tol)
        a.positions, a.residual = _ptr(out["positions"]), _ptr(out["residual"])
        a.iterations, a.status = _ptr(out["iterations"]), _ptr(out["status"])
        opts = make_opts(None, window_deform, True, False)
        cp = P.c_params()
        _lib.check(_lib.load().nsb_deform_inverse(C.byref(cp), C.byref(opts), C.byref(s), C.byref(a), _stream()),
                   "nsb_deform_inverse")
    out["converged"] = out["status"] == _lib.INV_CONVERGED
    return out


def track_points(P: NativeParams, points: torch.Tensor, *, time_from: float, times_to: Sequence[float], window_deform=None,
                 max_iter: int = 20, tol: float = 1e-4) -> Dict[str, torch.Tensor]:
    """Follow observed points of the frame at `time_from` to the frames at `times_to` along the deformation field: the
    canonical target is c = p + offset(p) from deform_jacobian's own forward at time_from, then deform_inverse at each
    time with init = points.  Tracking to time_from itself returns the points bit for bit with 0 iterations.  Returns
    {"positions" [K,n,3], "residual" [K,n], "iterations" [K,n], "converged" [K,n]} for the K times.  A track follows the
    deformation's motion only: where the hash ensemble's blend moved the surface between frames, a tracked surface point
    sits off that frame's isosurface."""
    _check_newton(max_iter, tol, "track_points")
    points = _f32c(points).reshape(-1, 3)
    _need_cuda(points)
    n, dev = int(points.shape[0]), points.device
    off = deform_jacobian(P, window_deform=window_deform, positions=points,
                          sample_times=torch.full((n,), float(time_from), dtype=_F32, device=dev))["offsets"]
    targets = points + off
    res = [deform_inverse(P, targets, uniform_time=float(t), init=points, window_deform=window_deform, max_iter=max_iter,
                          tol=tol) for t in times_to]
    if not res:
        return {"positions": torch.empty((0, n, 3), dtype=_F32, device=dev), "residual": torch.empty((0, n), dtype=_F32, device=dev),
                "iterations": torch.empty((0, n), dtype=torch.int32, device=dev),
                "converged": torch.empty((0, n), dtype=torch.bool, device=dev)}
    return {k: torch.stack([r[k] for r in res]) for k in ("positions", "residual", "iterations", "converged")}


def _world_grad_scale(P: NativeParams):
    """Per-axis factor that turns d h0 / d(normalised position) into d h0 / d(world position): 1 / aabb extent."""
    a = P.aabb_list
    return [1.0 / (a[3 + k] - a[k]) for k in range(3)]


def _normals_launch(P: NativeParams, cp, opts, s, n_samples: int, dev, *, offsets=None, grad_scale=(1.0, 1.0, 1.0),
                    packed_info=None, weights=None, keep=None, observation: bool = False) -> Dict[str, torch.Tensor]:
    """nsb_normals_forward on filled nsb_samples: per-sample normals [n, 3], and with packed_info / weights the per-ray
    composite `ray_normals` [R, 3].  observation: apply the deformation Jacobian (needs offsets and, in opts, the
    deformation window)."""
    a = _lib.NormalsArgs()
    keep = list(keep or [])
    if observation:
        a.observation_space, a.loss_scale = 1, VJP_LOSS_SCALE
        a.deform_packed_t, a.deform_packed_pe_t = _ptr(P.deform_packed_t), _ptr(P.pe_t())
        a.vjp_scratch = _ptr(_workspace("normals_vjp", max(n_samples, 1) * 12, dev))
    if offsets is not None:
        offsets = _f32c(offsets).reshape(-1, 3)
        _need_cuda(offsets)
        a.offsets = _ptr(offsets); keep.append(offsets)
    for k in range(3):
        a.grad_scale[k] = float(grad_scale[k])
    out = {"normals": _rows(n_samples, (3,), _F32, dev)}
    a.normals = _ptr(out["normals"])
    if packed_info is not None:
        packed_info = packed_info.to(torch.int64).contiguous()
        weights = _f32c(weights).reshape(-1)
        _need_cuda(packed_info, weights)
        keep += [packed_info, weights]
        R = int(packed_info.shape[0])
        out["ray_normals"] = torch.zeros((R, 3), dtype=_F32, device=dev)
        a.packed_info, a.n_rays, a.weights, a.out_normals = _ptr(packed_info), R, _ptr(weights), _ptr(out["ray_normals"])
    if n_samples > 0:
        _lib.check(_lib.load().nsb_normals_forward(C.byref(cp), C.byref(opts), C.byref(s), C.byref(a), _stream()),
                   "nsb_normals_forward")
    return out


def field_normals(P: NativeParams, *, window_hash=None, offsets: Optional[torch.Tensor] = None,
                  origins=None, directions=None, ray_times=None, t_starts=None, t_ends=None, ray_indices=None,
                  positions=None, sample_times=None, sample_blend_codes=None, n_samples_dev: Optional[torch.Tensor] = None,
                  uniform_time: Optional[float] = None, line_gather: bool = False, world_space: bool = False,
                  packed_info: Optional[torch.Tensor] = None, weights: Optional[torch.Tensor] = None,
                  disable_initial: bool = True, soft_transition: bool = True, space: str = "canonical",
                  window_deform=None, sample_warp_codes: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """Surface normals of the density field (nsb_normals_forward), nerfstudio's Field.get_normals:
    n = -normalize(d h0 / d x), h0 = mlp_base output 0 before trunc_exp, x = the normalised hash-input position after the
    in-box selector (outside the box x = 0, and the normal is the gradient at the box origin).  Takes the sample keywords
    of field_forward plus the `offsets` a deformed evaluation produced (canonical-space normals: the deformation
    Jacobian is not applied).  world_space=True divides the gradient by the box extent per axis before normalising.
    With offsets, the tables are gathered as field_forward gathers them for the same call (blended frame table / timestep
    stack unless line_gather or per-sample blend codes).  With packed_info [R,2] and weights [n] also `ray_normals`
    [R,3] = sum_i w_i n_i / (|sum_i w_i n_i| + 1e-10).  Not differentiable.  Returns {"normals": [n,3], ...}.
    space="observation" (with offsets) applies the deformation Jacobian: the gradient with respect to the OBSERVED
    position, -normalize(s (g + J^T D^-1 g)), zero where the warped position leaves the box (s = 0).  It needs the
    `window_deform` of the evaluation that produced the offsets, and `sample_warp_codes` if that evaluation took them.
    Without offsets there is no deformation and both spaces are the same."""
    if space not in NORMAL_SPACES:
        raise ValueError(f"space must be one of {NORMAL_SPACES}, got {space!r}")
    keep: list = []
    s = _lib.Samples()
    n = _fill_samples(s, keep, origins=origins, directions=directions, ray_times=ray_times, t_starts=t_starts, t_ends=t_ends,
                      ray_indices=ray_indices, positions=positions, sample_times=sample_times,
                      sample_blend_codes=sample_blend_codes)
    dev = (origins if origins is not None else positions).device
    if sample_blend_codes is not None:
        assert tuple(sample_blend_codes.shape) == (n, 32)
    if n_samples_dev is not None:
        assert n_samples_dev.dtype == torch.int64 and n_samples_dev.is_cuda and n_samples_dev.numel() == 1
        s.n_samples_dev = _ptr(n_samples_dev); keep.append(n_samples_dev)
    frame = None
    if offsets is not None:
        frame = _blended_tables(P, uniform_time, window_hash, disable_initial, soft_transition, line_gather, sample_blend_codes)
    observation = space == "observation" and offsets is not None
    if observation and sample_warp_codes is not None:
        _fill_sample_code_bias(P, s, keep, sample_warp_codes, n, dev)
    opts = make_opts(window_hash, window_deform if observation else None, offsets is not None, False, disable_initial,
                     soft_transition)
    cp = P.c_params(inference=frame is not None, frame=frame)
    return _normals_launch(P, cp, opts, s, n, dev, offsets=offsets,
                           grad_scale=_world_grad_scale(P) if world_space else (1.0, 1.0, 1.0),
                           packed_info=packed_info, weights=weights, keep=keep, observation=observation)


def _blended_tables(P: NativeParams, uniform_time, window_hash, disable_initial, soft_transition, line_gather=False,
                    sample_blend_codes=None) -> Optional[torch.Tensor]:
    """The member-blended tables an inference call gathers: the frame table of `uniform_time` when every sample carries
    that time (the caller's promise, e.g. one camera frame), else the timestep stack.  None (the per-sample blend of the
    128 B table lines) for line_gather or per-sample blend codes."""
    if line_gather or sample_blend_codes is not None:
        return None
    if uniform_time is not None:
        return P.frame_table(uniform_time, window_hash, disable_initial, soft_transition)
    return P.timestep_tables(window_hash, disable_initial, soft_transition)


def _fill_samples(s, keep, *, origins=None, directions=None, ray_times=None, t_starts=None, t_ends=None, ray_indices=None,
                  positions=None, sample_times=None, sample_directions=None, sample_blend_codes=None):
    if origins is not None:
        origins, directions, t_starts, t_ends = map(_f32c, (origins, directions, t_starts, t_ends))
        ray_indices = ray_indices.detach().to(torch.int32).contiguous()
        ray_times = None if ray_times is None else _f32c(ray_times).reshape(-1)
        _need_cuda(origins, directions, t_starts, t_ends, ray_indices, ray_times)
        s.origins, s.directions, s.ray_times = _ptr(origins), _ptr(directions), _ptr(ray_times)
        s.t_starts, s.t_ends, s.ray_indices = _ptr(t_starts), _ptr(t_ends), _ptr(ray_indices)
        keep += [origins, directions, t_starts, t_ends, ray_indices, ray_times]
        s.n_samples = int(t_starts.shape[0])
    else:
        positions = _f32c(positions).reshape(-1, 3)
        sample_times = None if sample_times is None else _f32c(sample_times).reshape(-1)
        sample_directions = None if sample_directions is None else _f32c(sample_directions).reshape(-1, 3)
        _need_cuda(positions, sample_times, sample_directions)
        s.positions, s.sample_times, s.sample_directions = _ptr(positions), _ptr(sample_times), _ptr(sample_directions)
        keep += [positions, sample_times, sample_directions]
        s.n_samples = int(positions.shape[0])
    if sample_blend_codes is not None:
        sample_blend_codes = _f32c(sample_blend_codes)
        s.sample_blend_codes = _ptr(sample_blend_codes); keep.append(sample_blend_codes)
    return s.n_samples


def field_backward(P: NativeParams, saved: Dict[str, torch.Tensor], d_sigma: Optional[torch.Tensor],
                   d_rgb: Optional[torch.Tensor], *, window_hash=None, loss_scale: float = 128.0,
                   want_tables: bool = True, want_codes: bool = True, want_dx: bool = False, rank1: bool = True,
                   defer_tables: bool = False, disable_initial=True, soft_transition=True,
                   **sample_kw) -> Dict[str, torch.Tensor]:
    """Backward of the density/colour MLPs and the hash ensemble (nsb_field_backward).
    saved: feat, xs, sigma, rgb from field_forward(want=(..., "feat", "xs")).  Returns fp32 gradients:
    d_base_w [3072], d_head_w [7168] (tcnn flat layouts), d_tables [entries,32,2], d_blend_codes [T,32], d_feat.
    With sample_blend_codes (per-sample conditioning, component API) the code gradient is d_sample_blend_codes [n,32]
    instead of d_blend_codes, and the table gradient takes the direct scatter."""
    lib = _lib.load()
    keep = []
    s = _lib.Samples()
    n = _fill_samples(s, keep, **sample_kw)
    dev = saved["feat"].device
    a = _lib.FieldBwdArgs()
    feat = saved["feat"].contiguous(); xs = _f32c(saved["xs"]); sg = _f32c(saved["sigma"]); cc = _f32c(saved.get("rgb"))
    dsg = None if d_sigma is None else _f32c(d_sigma).reshape(-1)
    drg = None if d_rgb is None else _f32c(d_rgb).reshape(-1, 3)
    _need_cuda(feat, xs, sg, cc, dsg, drg)
    a.field_packed_t = _ptr(P.field_packed_t)
    a.feat, a.xs, a.sigma, a.rgb, a.d_sigma, a.d_rgb = _ptr(feat), _ptr(xs), _ptr(sg), _ptr(cc), _ptr(dsg), _ptr(drg)
    a.loss_scale = float(loss_scale)
    if saved.get("corner_vals") is not None:
        a.corner_vals = _ptr(saved["corner_vals"])
    out = {"d_feat": _rows(n, (32,), _F32, dev, zero=True),
           "d_base_w": torch.zeros((3072,), dtype=_F32, device=dev), "d_head_w": torch.zeros((7168,), dtype=_F32, device=dev)}
    a.d_feat, a.d_base_w, a.d_head_w = _ptr(out["d_feat"]), _ptr(out["d_base_w"]), _ptr(out["d_head_w"])
    # defer_tables: leave the table gradient in its rank-1 form (out["pending"]) for table_adam_step / rank1_expand
    # instead of expanding it to a dense 1.6 GB tensor here; falls back to dense when the rank-1 path is unavailable.
    slot, n_slots = _rank1_slots(P, dev, sample_kw) if (rank1 and (want_tables or want_codes)) else (None, 0)
    defer = bool(defer_tables and want_tables and slot is not None)
    if want_tables and not defer:
        out["d_tables"] = torch.zeros((P.levels["total_entries"], 32, 2), dtype=_F32, device=dev)
        a.d_tables = _ptr(out["d_tables"])
    if want_codes and sample_kw.get("sample_blend_codes") is not None:
        out["d_sample_blend_codes"] = _rows(n, (32,), _F32, dev)     # written for every sample by the kernel
        a.d_sample_blend_codes = _ptr(out["d_sample_blend_codes"])
    elif want_codes:
        out["d_blend_codes"] = torch.zeros((P.n_timesteps, 32), dtype=_F32, device=dev)
        a.d_blend_codes = _ptr(out["d_blend_codes"])
    if want_dx:
        out["d_xs"] = _rows(n, (3,), _F32, dev, zero=True)
        a.d_xs = _ptr(out["d_xs"])
    if n == 0:
        return out
    if slot is not None:
        g1 = torch.zeros((n_slots, P.levels["total_entries"], 2), dtype=_F32, device=dev)
        a.g_rank1, a.ts_slot, a.n_slots = _ptr(g1), _ptr(slot), n_slots
        keep += [g1, slot]
        if defer:
            cw = torch.zeros((n_slots, 32), dtype=_F32, device=dev)
            a.cw_slots_out = _ptr(cw)
            out["pending"] = {"g_rank1": g1, "cw_slots": cw, "n_slots": n_slots,
                              "slots_are_timesteps": P.n_timesteps <= 32}
    opts = make_opts(window_hash, None, False, True, disable_initial, soft_transition)
    cp = P.c_params()
    _lib.check(lib.nsb_field_backward(C.byref(cp), C.byref(opts), C.byref(s), C.byref(a), _stream()), "nsb_field_backward")
    return out


def _rank1_slots(P: "NativeParams", dev, sample_kw):
    """Timestep -> slot map of the rank-1 table-gradient scatter (32x fewer atomics than the direct one): needs
    table-indexed blend codes and <= 32 distinct timesteps in the batch.  Returns (slot [T] int32 | None, n_slots)."""
    if sample_kw.get("sample_blend_codes") is not None:
        return None, 0
    T = P.n_timesteps
    if T <= 32:
        return torch.arange(T, dtype=torch.int32, device=dev), T
    tt = sample_kw.get("ray_times") if sample_kw.get("origins") is not None else sample_kw.get("sample_times")
    if tt is None:
        return None, 0
    ts_idx = (tt.reshape(-1).float() * (T - 1)).round().clamp_(0, T - 1).long()
    uniq = torch.unique(ts_idx)                       # host sync: the slot count is data dependent
    if uniq.numel() > 32:
        return None, 0
    slot = torch.full((T,), -1, dtype=torch.int32, device=dev)
    slot[uniq] = torch.arange(uniq.numel(), dtype=torch.int32, device=dev)
    return slot, int(uniq.numel())


def table_adam_step(tables: torch.Tensor, exp_avg: torch.Tensor, exp_avg_sq: torch.Tensor,
                    tables_half: Optional[torch.Tensor], *, step: int, lr: float, betas=(0.9, 0.999), eps: float = 1e-8,
                    weight_decay: float = 0.0, grad: Optional[torch.Tensor] = None, pending: Optional[dict] = None,
                    grad_scale: float = 1.0) -> None:
    """torch.optim.Adam's update of the native fp32 table [E,32,2] in one fused pass (nsb_table_adam_step): the gradient
    is a dense tensor and/or the deferred rank-1 form from field_backward(defer_tables=True); the fp16 copy the forward
    kernels read is rewritten in the same pass.  In place; `step` is the 1-based step count."""
    lib = _lib.load()
    _need_cuda(tables, exp_avg, exp_avg_sq, tables_half, grad)
    for t in (tables, exp_avg, exp_avg_sq):
        assert t.dtype == _F32 and t.is_contiguous() and t.shape == tables.shape
    a = _lib.TableAdamArgs()
    a.total_entries = tables.shape[0]
    a.tables, a.exp_avg, a.exp_avg_sq = _ptr(tables), _ptr(exp_avg), _ptr(exp_avg_sq)
    if tables_half is not None:
        assert tables_half.dtype == torch.float16 and tables_half.is_contiguous() and tables_half.shape == tables.shape
        a.tables_half = _ptr(tables_half)
    if grad is not None:
        assert grad.dtype == _F32 and grad.is_contiguous() and grad.shape == tables.shape
        a.grad = _ptr(grad)
    if pending is not None:
        a.g_rank1, a.cw_slots, a.n_slots = _ptr(pending["g_rank1"]), _ptr(pending["cw_slots"]), int(pending["n_slots"])
    a.grad_scale = float(grad_scale)
    a.lr, a.beta1, a.beta2, a.eps, a.weight_decay = float(lr), float(betas[0]), float(betas[1]), float(eps), float(weight_decay)
    bc1, bc2 = 1.0 - float(betas[0]) ** step, 1.0 - float(betas[1]) ** step
    a.bias_correction1, a.bias_correction2 = bc1, bc2
    # the scalars exactly as torch.optim.Adam (_multi_tensor_adam) forms them: Python doubles, rounded once to float
    a.step_size, a.bias_correction2_sqrt = float(lr) / bc1, bc2 ** 0.5
    a.one_minus_beta1, a.one_minus_beta2 = 1.0 - float(betas[0]), 1.0 - float(betas[1])
    _lib.check(lib.nsb_table_adam_step(C.byref(a), _stream()), "nsb_table_adam_step")


def rank1_expand(pending: dict, total_entries: int, grad_scale: float = 1.0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Dense fp32 table gradient [E,32,2] (+= into `out`) from the deferred rank-1 form (nsb_rank1_expand)."""
    lib = _lib.load()
    g1 = pending["g_rank1"]
    if out is None:
        out = torch.zeros((total_entries, 32, 2), dtype=_F32, device=g1.device)
    _need_cuda(g1, out)
    _lib.check(lib.nsb_rank1_expand(_ptr(g1), _ptr(pending["cw_slots"]), int(pending["n_slots"]), int(total_entries),
                                    float(grad_scale), _ptr(out), _stream()), "nsb_rank1_expand")
    return out


LOSS_NAMES = ("rgb_loss", "alpha_loss", "empty_loss", "near_loss", "depth_loss", "dist_loss")


def _loss_args(packed_info, t_starts, t_ends, weights, rgb, acc, depth, image, alpha, depth_target, cfg: dict, keep: list):
    a = _lib.LossArgs()
    pi = packed_info.to(torch.int64).contiguous()
    ts, te, w = _f32c(t_starts).reshape(-1), _f32c(t_ends).reshape(-1), _f32c(weights).reshape(-1)
    rgb_, acc_, dep_ = _f32c(rgb).reshape(-1, 3), _f32c(acc).reshape(-1), _f32c(depth).reshape(-1)
    img = _f32c(image).reshape(-1, 3)
    al = None if alpha is None else _f32c(alpha).reshape(-1)
    dt = None if depth_target is None else _f32c(depth_target).reshape(-1)
    _need_cuda(pi, ts, te, w, rgb_, acc_, dep_, img, al, dt)
    keep += [pi, ts, te, w, rgb_, acc_, dep_, img, al, dt]
    a.n_rays, a.n_samples = int(pi.shape[0]), int(w.shape[0])
    a.packed_info, a.t_starts, a.t_ends, a.weights = _ptr(pi), _ptr(ts), _ptr(te), _ptr(w)
    a.rgb, a.acc, a.depth, a.image, a.alpha, a.depth_target = _ptr(rgb_), _ptr(acc_), _ptr(dep_), _ptr(img), _ptr(al), _ptr(dt)
    a.use_masked_rgb = int(bool(cfg.get("use_masked_rgb", True)))
    a.alpha_mask_threshold = float(cfg.get("alpha_mask_threshold", 0.0))
    for k in ("lambda_alpha", "lambda_empty", "lambda_near", "lambda_depth", "lambda_dist"):
        setattr(a, k, float(cfg.get(k) or 0.0))
    a.eps_depth = float(cfg.get("eps_depth", 0.0))
    a.dist_max_rays = int(cfg.get("dist_max_rays", 1 << 62))
    return a


def losses_forward(packed_info, t_starts, t_ends, weights, rgb, acc, depth, image, alpha, depth_target, cfg: dict):
    """The six losses of models/base.py in two launches (nsb_losses_forward).  Returns (values [6] in LOSS_NAMES order,
    state for losses_backward).  cfg: use_masked_rgb, alpha_mask_threshold, lambda_{alpha,empty,near,depth,dist},
    eps_depth, dist_max_rays; a lambda of 0 / a missing alpha or depth_target switches a term off (value 0)."""
    lib = _lib.load()
    keep: list = []
    a = _loss_args(packed_info, t_starts, t_ends, weights, rgb, acc, depth, image, alpha, depth_target, cfg, keep)
    dev = keep[0].device
    accum = torch.empty(16, dtype=torch.float64, device=dev)
    values = torch.empty(6, dtype=_F32, device=dev)
    coef = torch.empty(8, dtype=_F32, device=dev)
    a.accum, a.values, a.coef = _ptr(accum), _ptr(values), _ptr(coef)
    _lib.check(lib.nsb_losses_forward(C.byref(a), _stream()), "nsb_losses_forward")
    return values, {"args": a, "keep": keep + [accum, values, coef]}


def losses_backward(state: dict, upstream: torch.Tensor):
    """Gradients of sum_k upstream[k] * values[k] w.r.t. (rgb [R,3], acc [R], depth [R], weights [S])."""
    lib = _lib.load()
    a, keep = state["args"], state["keep"]
    dev = keep[0].device
    up = _f32c(upstream).reshape(6)
    d_rgb = torch.empty((a.n_rays, 3), dtype=_F32, device=dev)
    d_acc = torch.empty((a.n_rays,), dtype=_F32, device=dev)
    d_depth = torch.empty((a.n_rays,), dtype=_F32, device=dev)
    d_w = _rows(a.n_samples, (), _F32, dev, zero=True)
    a.upstream, a.d_rgb, a.d_acc, a.d_depth, a.d_weights = _ptr(up), _ptr(d_rgb), _ptr(d_acc), _ptr(d_depth), _ptr(d_w)
    _lib.check(lib.nsb_losses_backward(C.byref(a), _stream()), "nsb_losses_backward")
    return d_rgb, d_acc, d_depth, d_w


def deform_backward(P: NativeParams, saved: Dict[str, torch.Tensor], d_xs: torch.Tensor, *, window_deform=None,
                    loss_scale: float = 128.0, sample_warp_codes: Optional[torch.Tensor] = None,
                    **sample_kw) -> Dict[str, torch.Tensor]:
    """Backward of the SE(3) deformation field (nsb_deform_backward).  saved: deform_acts, deform_enc from
    field_forward(want=(..., "deform_acts")); d_xs from field_backward(want_dx=True).  Returns fp32 gradients in
    the reference layouts: d_stem_w (list of 6), d_stem_b [6,128], d_r_w, d_r_b, d_v_w, d_v_b, d_warp_codes [T,128].
    sample_warp_codes [n,128]: the per-sample codes the forward was given (component API); the code gradient is then
    d_sample_warp_codes [n,128] instead of d_warp_codes."""
    lib = _lib.load()
    keep = []
    s = _lib.Samples()
    n = _fill_samples(s, keep, **sample_kw)
    dev = d_xs.device
    a = _lib.DeformBwdArgs()
    dxs = _f32c(d_xs).reshape(-1, 3)
    _need_cuda(dxs, sample_warp_codes)
    a.deform_packed_t = _ptr(P.deform_packed_t)
    a.deform_acts, a.deform_enc, a.d_xs = _ptr(saved["deform_acts"]), _ptr(saved["deform_enc"]), _ptr(dxs)
    a.loss_scale = float(loss_scale)
    dims = [(128, 173), (128, 128), (128, 128), (128, 128), (128, 301), (128, 128)]
    out = {"d_stem_w": [torch.zeros(d, dtype=_F32, device=dev) for d in dims],
           "d_stem_b": torch.zeros((6, 128), dtype=_F32, device=dev),
           "d_r_w": torch.zeros((3, 128), dtype=_F32, device=dev), "d_r_b": torch.zeros((3,), dtype=_F32, device=dev),
           "d_v_w": torch.zeros((3, 128), dtype=_F32, device=dev), "d_v_b": torch.zeros((3,), dtype=_F32, device=dev)}
    for l in range(6):
        a.d_stem_w[l] = _ptr(out["d_stem_w"][l])
    a.d_stem_b, a.d_r_w, a.d_r_b = _ptr(out["d_stem_b"]), _ptr(out["d_r_w"]), _ptr(out["d_r_b"])
    a.d_v_w, a.d_v_b = _ptr(out["d_v_w"]), _ptr(out["d_v_b"])
    if sample_warp_codes is not None:
        assert sample_warp_codes.shape == (n, 128)
        swc = sample_warp_codes.detach().to(torch.float16).contiguous()      # the fp16 operand the forward used
        keep.append(swc)
        out["d_sample_warp_codes"] = _rows(n, (128,), _F32, dev, zero=True)
        a.sample_warp_codes, a.d_sample_warp_codes = _ptr(swc), _ptr(out["d_sample_warp_codes"])
    else:
        out["d_warp_codes"] = torch.zeros((P.n_timesteps, 128), dtype=_F32, device=dev)
        a.d_warp_codes = _ptr(out["d_warp_codes"])
    ws = _workspace("deform_bwd", int(lib.nsb_deform_bwd_workspace_bytes()), dev)
    a.dw_workspace = _ptr(ws)
    if n == 0:
        return out
    opts = make_opts(None, window_deform, True, False)
    cp = P.c_params()
    _lib.check(lib.nsb_deform_backward(C.byref(cp), C.byref(opts), C.byref(s), C.byref(a), _stream()), "nsb_deform_backward")
    return out


def hash_blend_forward(P: NativeParams, x: torch.Tensor, codes: torch.Tensor, window_hash=None,
                       out_half: bool = True, disable_initial=True, soft_transition=True) -> torch.Tensor:
    """HashEnsemble.forward (hash_ensemble.py:93-158): x [n,3] in [0,1), codes [n,32]."""
    lib = _lib.load()
    x = _f32c(x); codes = _f32c(codes)
    _need_cuda(x, codes)
    n = x.shape[0]
    out = torch.empty((n, 32), dtype=torch.float16 if out_half else _F32, device=x.device)
    if n == 0:
        return out
    opts = make_opts(window_hash, None, False, False, disable_initial, soft_transition)
    cp = P.c_params()
    rc = lib.nsb_hash_blend_forward(C.byref(cp), C.byref(opts), _ptr(x), _ptr(codes), n, _ptr(out), int(out_half), _stream())
    _lib.check(rc, "nsb_hash_blend_forward")
    return out


def hash_blend_backward(P: NativeParams, x: torch.Tensor, codes: torch.Tensor, d_out: torch.Tensor, window_hash=None,
                        want_tables: bool = True, want_codes: bool = True, want_dx: bool = True, disable_initial=True,
                        soft_transition=True) -> Dict[str, torch.Tensor]:
    """Backward of hash_blend_forward (nsb_hash_blend_backward) for d_out [n,32]: fp32 d_tables [entries,32,2] (dense),
    d_codes [n,32], d_x [n,3] -- each only when wanted."""
    lib = _lib.load()
    x = _f32c(x); codes = _f32c(codes); d_out = _f32c(d_out)
    _need_cuda(x, codes, d_out)
    n, dev = x.shape[0], x.device
    assert codes.shape == (n, 32) and d_out.shape == (n, 32)
    out = {}
    if want_tables:
        out["d_tables"] = torch.zeros((P.levels["total_entries"], 32, 2), dtype=_F32, device=dev)
    if want_codes:
        out["d_codes"] = torch.empty((n, 32), dtype=_F32, device=dev)
    if want_dx:
        out["d_x"] = torch.empty((n, 3), dtype=_F32, device=dev)
    if n == 0:
        return out
    opts = make_opts(window_hash, None, False, False, disable_initial, soft_transition)
    cp = P.c_params()
    rc = lib.nsb_hash_blend_backward(C.byref(cp), C.byref(opts), _ptr(x), _ptr(codes), n, _ptr(d_out),
                                     _ptr(out.get("d_tables")), _ptr(out.get("d_codes")), _ptr(out.get("d_x")), _stream())
    _lib.check(rc, "nsb_hash_blend_backward")
    return out


def composite(packed_info: torch.Tensor, t_starts, t_ends, sigma, rgb, offsets=None, training=False,
              want_weights=True) -> Dict[str, torch.Tensor]:
    """render_weight_from_density + RGB(white)/Depth(expected)/Accumulation/Deformation renderers."""
    lib = _lib.load()
    _need_cuda(packed_info, t_starts, t_ends, sigma, rgb, offsets)
    packed_info = packed_info.to(torch.int64).contiguous()
    R = packed_info.shape[0]; n = t_starts.shape[0]; dev = t_starts.device
    a = _lib.CompositeArgs()
    a.n_rays, a.n_samples = R, n
    a.packed_info = _ptr(packed_info)
    ts, te, sg, cc = map(_f32c, (t_starts, t_ends, sigma, rgb))
    off = _f32c(offsets)
    a.t_starts, a.t_ends, a.sigma, a.rgb, a.offsets = _ptr(ts), _ptr(te), _ptr(sg), _ptr(cc), _ptr(off)
    a.training = int(training)
    out = {"rgb": torch.empty((R, 3), dtype=_F32, device=dev), "accumulation": torch.empty((R, 1), dtype=_F32, device=dev),
           "depth": torch.empty((R, 1), dtype=_F32, device=dev)}
    a.out_rgb, a.out_acc, a.out_depth = _ptr(out["rgb"]), _ptr(out["accumulation"]), _ptr(out["depth"])
    if off is not None:
        out["deformation"] = torch.empty((R, 3), dtype=_F32, device=dev); a.out_deform = _ptr(out["deformation"])
    if want_weights:
        out["weights"] = _rows(n, (1,), _F32, dev); a.out_weights = _ptr(out["weights"])
    ws = torch.empty((2,), dtype=torch.int32, device=dev)
    a.workspace = _ptr(ws)
    rc = lib.nsb_composite_forward(C.byref(a), _stream())
    _lib.check(rc, "nsb_composite_forward")
    out["workspace"] = ws
    return out


def composite_backward(packed_info, t_starts, t_ends, sigma, rgb, workspace, d_out_rgb, d_out_acc=None, d_out_depth=None,
                       d_weights=None):
    """Backward of composite() in training mode -> (d_sigma [S], d_rgb [S,3])."""
    lib = _lib.load()
    packed_info = packed_info.to(torch.int64).contiguous()
    ts, te, sg, cc = map(_f32c, (t_starts, t_ends, sigma, rgb))
    g_rgb = _f32c(d_out_rgb).reshape(-1, 3)
    g_acc = None if d_out_acc is None else _f32c(d_out_acc).reshape(-1)
    g_dep = None if d_out_depth is None else _f32c(d_out_depth).reshape(-1)
    g_w = None if d_weights is None else _f32c(d_weights).reshape(-1)
    _need_cuda(packed_info, ts, te, sg, cc, g_rgb, g_acc, g_dep, g_w, workspace)
    R, n = packed_info.shape[0], ts.shape[0]
    a = _lib.CompositeBwdArgs()
    a.n_rays, a.n_samples, a.packed_info = R, n, _ptr(packed_info)
    a.t_starts, a.t_ends, a.sigma, a.rgb = _ptr(ts), _ptr(te), _ptr(sg), _ptr(cc)
    a.d_out_rgb, a.d_out_acc, a.d_out_depth, a.d_weights = _ptr(g_rgb), _ptr(g_acc), _ptr(g_dep), _ptr(g_w)
    a.workspace = _ptr(workspace)
    d_sigma = _rows(n, (), _F32, ts.device, zero=True)
    d_rgb = _rows(n, (3,), _F32, ts.device, zero=True)
    a.d_sigma, a.d_rgb = _ptr(d_sigma), _ptr(d_rgb)
    _lib.check(lib.nsb_composite_backward(C.byref(a), _stream()), "nsb_composite_backward")
    return d_sigma, d_rgb


def march_fixed(origins, directions, aabb: torch.Tensor, n_per_ray: int, step: float, near_plane: float = 0.0):
    lib = _lib.load()
    origins, directions = _f32c(origins), _f32c(directions)
    _need_cuda(origins, directions)
    dev = origins.device
    R = origins.shape[0]
    aabb_d = aabb.detach().to(dev, _F32).reshape(-1).contiguous()
    n = R * n_per_ray
    ts, te = _rows(n, (), _F32, dev), _rows(n, (), _F32, dev)
    ri = _rows(n, (), torch.int32, dev)
    info = torch.empty((R, 2), dtype=torch.int64, device=dev)
    rc = lib.nsb_march_fixed(_ptr(origins), _ptr(directions), R, _ptr(aabb_d), n_per_ray, float(step), float(near_plane),
                             _ptr(ts), _ptr(te), _ptr(ri), _ptr(info), _stream())
    _lib.check(rc, "nsb_march_fixed")
    return ts, te, ri, info


def march_occupancy(origins, directions, near_planes, far_planes, binaries: torch.Tensor, aabbs: torch.Tensor,
                    step: float, cone_angle: float = 0.0):
    """nerfacc traverse_grids: two passes (count, exclusive scan, fill).  Returns packed
    (t_starts, t_ends, ray_indices int32, packed_info int64 [R,2])."""
    lib = _lib.load()
    origins, directions, near_planes, far_planes = map(_f32c, (origins, directions, near_planes, far_planes))
    _need_cuda(origins, directions, near_planes, far_planes, binaries, aabbs)
    dev = origins.device
    R = origins.shape[0]
    b8 = binaries.detach().to(torch.uint8).contiguous()
    levels, res = int(b8.shape[0]), int(b8.shape[1])
    assert b8.shape[1] == b8.shape[2] == b8.shape[3], "cubic grids only"
    ab = aabbs.detach().to(dev, _F32).reshape(levels, 6).contiguous()
    a = _lib.MarchArgs()
    a.n_rays = R
    a.origins, a.directions, a.near_planes, a.far_planes = _ptr(origins), _ptr(directions), _ptr(near_planes), _ptr(far_planes)
    a.binaries, a.aabbs, a.levels, a.res = _ptr(b8), _ptr(ab), levels, res
    a.step, a.cone_angle = float(step), float(cone_angle)
    counts = torch.empty((R,), dtype=torch.int32, device=dev)
    a.counts = _ptr(counts)
    _lib.check(lib.nsb_march_occupancy(C.byref(a), _stream()), "nsb_march_occupancy(count)")
    cnt64 = counts.to(torch.int64)
    incl = torch.cumsum(cnt64, 0)
    offsets = (incl - cnt64).contiguous()
    n = int(incl[-1].item()) if R > 0 else 0       # host sync: the packed size is data dependent
    ts, te = _rows(n, (), _F32, dev), _rows(n, (), _F32, dev)
    ri = _rows(n, (), torch.int32, dev)
    if n > 0:
        a.offsets, a.t_starts, a.t_ends, a.ray_indices = _ptr(offsets), _ptr(ts), _ptr(te), _ptr(ri)
        _lib.check(lib.nsb_march_occupancy(C.byref(a), _stream()), "nsb_march_occupancy(fill)")
    return ts, te, ri, torch.stack([offsets, cnt64], -1)


def visibility_mask(packed_info, t_starts, t_ends, sigma, early_stop_eps: float, alpha_thre: float):
    lib = _lib.load()
    _need_cuda(packed_info, t_starts, t_ends, sigma)
    packed_info = packed_info.to(torch.int64).contiguous()
    ts, te, sg = map(_f32c, (t_starts, t_ends, sigma))
    R = packed_info.shape[0]; n = ts.shape[0]
    mask = _rows(n, (), torch.uint8, ts.device, zero=True)
    kept = torch.zeros((R,), dtype=torch.int32, device=ts.device)
    rc = lib.nsb_visibility_mask(_ptr(packed_info), R, _ptr(ts), _ptr(te), _ptr(sg), float(early_stop_eps),
                                 float(alpha_thre), _ptr(mask), _ptr(kept), _stream())
    _lib.check(rc, "nsb_visibility_mask")
    return mask.bool(), kept


def occ_update(occs: torch.Tensor, binaries: torch.Tensor, cell_ids: torch.Tensor, occ_new: torch.Tensor,
               ema_decay: float, occ_thre: float) -> None:
    """nerfacc OccGridEstimator._update's EMA-max + re-threshold, in place (nsb_occ_update): `occs` float [n_cells],
    `binaries` bool (any shape with n_cells elements); duplicates in cell_ids resolve to the largest candidate."""
    lib = _lib.load()
    _need_cuda(occs, binaries, cell_ids, occ_new)
    assert occs.dtype == _F32 and occs.is_contiguous() and binaries.dtype == torch.bool and binaries.is_contiguous()
    assert binaries.numel() == occs.numel()
    ids = cell_ids.detach().to(torch.int64).contiguous()
    new = _f32c(occ_new).reshape(-1)
    assert ids.shape == new.shape
    n_cells = occs.numel()
    ws = _workspace("occ_update", int(lib.nsb_occ_update_scratch_bytes(n_cells)), occs.device)
    _lib.check(lib.nsb_occ_update(_ptr(occs), _ptr(binaries), n_cells, _ptr(ids), _ptr(new), int(ids.numel()),
                                  float(ema_decay), float(occ_thre), _ptr(ws), _stream()), "nsb_occ_update")


def march_occupancy_packed(origins, directions, near_planes, far_planes, binaries: torch.Tensor, aabbs: torch.Tensor,
                           step: float, cone_angle: float = 0.0, capacity: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """nerfacc traverse_grids as ONE cooperative launch without host synchronisation (nsb_march_occupancy_packed): the
    samples land in arrays of `capacity` slots (default: an upper bound of the march), the count stays on the device.
    Returns t_starts / t_ends / ray_indices [capacity], packed_info [R,2], `n_total` (int64 device scalar), `header`."""
    lib = _lib.load()
    origins, directions, near_planes, far_planes = map(_f32c, (origins, directions, near_planes, far_planes))
    _need_cuda(origins, directions, near_planes, far_planes, binaries, aabbs)
    dev, R = origins.device, int(origins.shape[0])
    b8 = binaries.detach().contiguous()
    b8 = b8.view(torch.uint8) if b8.dtype == torch.bool else b8.to(torch.uint8)
    levels, res = int(b8.shape[0]), int(b8.shape[1])
    assert b8.shape[1] == b8.shape[2] == b8.shape[3], "cubic grids only"
    ab = aabbs.detach().to(dev, _F32).reshape(levels, 6).contiguous()
    if capacity is None:
        diag = float((ab[:, 3:] - ab[:, :3]).norm(dim=-1).max())
        capacity = R * (int(diag / float(step)) + 2 * levels + 2)
    cap = max(int(capacity), 1)
    a = _lib.MarchArgs()
    a.n_rays = R
    a.origins, a.directions, a.near_planes, a.far_planes = _ptr(origins), _ptr(directions), _ptr(near_planes), _ptr(far_planes)
    a.binaries, a.aabbs, a.levels, a.res = _ptr(b8), _ptr(ab), levels, res
    a.step, a.cone_angle = float(step), float(cone_angle)
    out = {"t_starts": torch.empty((cap,), dtype=_F32, device=dev), "t_ends": torch.empty((cap,), dtype=_F32, device=dev),
           "ray_indices": torch.empty((cap,), dtype=torch.int32, device=dev),
           "packed_info": torch.empty((R, 2), dtype=torch.int64, device=dev), "capacity": cap}
    a.t_starts, a.t_ends, a.ray_indices = _ptr(out["t_starts"]), _ptr(out["t_ends"]), _ptr(out["ray_indices"])
    ws = torch.empty((int(lib.nsb_render_workspace_bytes(R)) + 7) // 8, dtype=torch.int64, device=dev)
    scratch = torch.empty((2, cap), dtype=_F32, device=dev) if cap >= R else None
    out["header"], out["n_total"] = ws, ws[2:3]
    out["_keep"] = [origins, directions, near_planes, far_planes, b8, ab, scratch]
    if R > 0:
        _lib.check(lib.nsb_march_occupancy_packed(C.byref(a), cap, _ptr(out["packed_info"]), _ptr(ws), _ptr(scratch), _stream()),
                   "nsb_march_occupancy_packed")
    else:
        ws.zero_()
    return out


def visibility_compact(cand: Dict[str, torch.Tensor], sigma: torch.Tensor, early_stop_eps: float, alpha_thre: float,
                       alpha_thre_cap: Optional[torch.Tensor] = None, payload: Optional[Dict[str, torch.Tensor]] = None
                       ) -> Dict[str, torch.Tensor]:
    """nerfacc render_visibility_from_density + packing of the surviving samples, one cooperative launch, no host sync
    (nsb_visibility_compact).  cand: march_occupancy_packed's result; sigma [capacity]; alpha_thre_cap: device scalar
    (occs.mean()) -> alpha_thre = min(alpha_thre, cap).  payload: optional {feat [cap,32] half, xs [cap,4], corner_vals
    [cap,16,8,2] half} rows that move with their samples.  Returns the packed arrays [capacity], packed_info, n_total."""
    lib = _lib.load()
    dev = sigma.device
    cap, R = int(cand["capacity"]), int(cand["packed_info"].shape[0])
    sg = _f32c(sigma).reshape(-1)
    assert sg.shape[0] >= cap
    a = _lib.VisCompactArgs()
    a.n_rays, a.capacity = R, cap
    a.packed_info, a.t_starts, a.t_ends, a.sigma, a.ray_indices = (_ptr(cand["packed_info"]), _ptr(cand["t_starts"]), _ptr(cand["t_ends"]),
                                                                   _ptr(sg), _ptr(cand["ray_indices"]))
    a.early_stop_eps, a.alpha_thre = float(early_stop_eps), float(alpha_thre)
    keep = [sg]
    if alpha_thre_cap is not None:
        capt = _f32c(alpha_thre_cap).reshape(1)
        a.alpha_thre_cap = _ptr(capt); keep.append(capt)
    out = {"t_starts": torch.empty((cap,), dtype=_F32, device=dev), "t_ends": torch.empty((cap,), dtype=_F32, device=dev),
           "ray_indices": torch.empty((cap,), dtype=torch.int32, device=dev),
           "packed_info": torch.empty((R, 2), dtype=torch.int64, device=dev), "capacity": cap}
    a.out_packed_info, a.out_t_starts, a.out_t_ends, a.out_ray_indices = (_ptr(out["packed_info"]), _ptr(out["t_starts"]),
                                                                          _ptr(out["t_ends"]), _ptr(out["ray_indices"]))
    if payload:
        for name, shape, dt in (("feat", (cap, 32), torch.float16), ("xs", (cap, 4), _F32), ("corner_vals", (cap, 16, 8, 2), torch.float16)):
            if payload.get(name) is not None:
                src = payload[name]
                assert src.dtype == dt and src.is_contiguous() and tuple(src.shape) == shape, (name, src.shape, src.dtype)
                out[name] = torch.empty(shape, dtype=dt, device=dev)
                setattr(a, name, _ptr(src)); setattr(a, "out_" + name, _ptr(out[name])); keep.append(src)
    ws = torch.empty((int(lib.nsb_vis_compact_workspace_bytes(R, cap)) + 7) // 8, dtype=torch.int64, device=dev)
    a.workspace = _ptr(ws)
    out["header"], out["n_total"] = ws, ws[2:3]
    out["_keep"] = keep + [cand]
    if R > 0:
        _lib.check(lib.nsb_visibility_compact(C.byref(a), _stream()), "nsb_visibility_compact")
    else:
        ws.zero_()
    return out


class RenderResult(dict):
    """Per-ray outputs of render_rays plus lazy access to the packed per-sample arrays (`packed()` synchronises once)."""

    def packed(self) -> Dict[str, torch.Tensor]:
        b = self["_buffers"]
        h = b["header"][:3].tolist()                  # the ONE host synchronisation, only when asked for
        n, status = int(h[2]), int(h[1]) >> 32
        if status != 0 or n > b["capacity"]:
            raise RuntimeError(f"render_rays: the march produced more samples than the workspace holds "
                               f"(n_total {n}, capacity {b['capacity']}, status {status}); pass a larger capacity")
        out = {k: b[k][:n] for k in ("t_starts", "t_ends", "ray_indices", "sigma", "rgb", "offsets", "weights", "normals")
               if b.get(k) is not None}
        out["weights"] = out["weights"][:, None]
        return out


def render_rays(P: NativeParams, origins, directions, ray_times, *, window_hash=None, window_deform=None,
                use_deformation=True, training=False, sampler: str = "occupancy", n_per_ray: int = 0,
                near_plane: float = 0.0, near_planes=None, far_planes=None, binaries=None, aabbs=None,
                step: float = 1e-3, cone_angle: float = 0.0, capacity: Optional[int] = None,
                disable_initial=True, soft_transition=True, single_traversal: bool = True,
                uniform_time: Optional[float] = None, line_gather: bool = False,
                want_normals: bool = False, normals_space: str = "canonical",
                time_interpolation: str = "nearest") -> RenderResult:
    """The fused inference render (nsb_render_forward): sampler -> field -> composite without a host synchronisation.
    sampler 'fixed' (n_per_ray steps from the box entry: ONE launch) or 'occupancy' (nerfacc march of `binaries`
    [levels,res,res,res] within per-ray near_planes / far_planes: the cooperative march launch + one fused launch;
    single_traversal=False: count | scan | fill instead of one traversal into per-ray slots + a packing copy).  Returns the per-ray outputs (rgb, accumulation,
    depth, deformation, num_samples_per_ray, packed_info); `.packed()` gives the per-sample arrays (one sync).
    capacity: per-sample workspace size; default = an upper bound of the march (rays x ceil(largest diagonal / step) + 2).
    The field gathers member-blended tables (frame_table for a uniform_time, timestep_tables otherwise) unless
    line_gather=True forces the per-sample blend of the 128 B table lines.
    want_normals=True adds `normals` [R,3]: the world-space surface normals of the call's own packed samples (field_normals
    on the same tables), composited with the render weights and normalised; still without a host synchronisation.
    normals_space="observation" applies the deformation Jacobian to them (field_normals(space=...)); without
    use_deformation both spaces are the same.
    time_interpolation="linear" renders at continuous times (DESIGN 4.2g) instead of rounding each time to the nearest
    timestep: with a uniform_time on the one-timestep view P.at_time(uniform_time) (any sampler, deformation and
    normals); with mixed ray_times on nsb_render_forward_interp (timestep stack or line gather, chosen as above), which
    needs use_deformation, the wgmma kernels and no normals.  Neither path synchronises with the host."""
    if normals_space not in NORMAL_SPACES:
        raise ValueError(f"normals_space must be one of {NORMAL_SPACES}, got {normals_space!r}")
    # the default ("nearest") costs one comparison: the host issues this call back to back in the render loop
    mixed_linear = (time_interpolation != "nearest" and _check_time_interpolation(time_interpolation, "render_rays")
                    and uniform_time is None)
    if mixed_linear:
        why = ("use_deformation=False" if not use_deformation else "want_normals=True" if want_normals else
               "the non-wgmma kernels (NSB_TCGEN05=0)" if (P.deform_packed_umma is None and getattr(P, "_umma_src", None) is None)
               else None)
        if why is not None:
            raise NotImplementedError(f"render_rays: time_interpolation='linear' with mixed ray times and {why}")
    elif time_interpolation == "linear":
        P = P.at_time(uniform_time)
    lib = _lib.load()
    origins, directions = _f32c(origins).reshape(-1, 3), _f32c(directions).reshape(-1, 3)
    ray_times = None if ray_times is None else _f32c(ray_times).reshape(-1)
    _need_cuda(origins, directions, ray_times, near_planes, far_planes, binaries)
    dev, R = origins.device, int(origins.shape[0])
    a = _lib.RenderArgs()
    keep = [origins, directions, ray_times]
    a.n_rays, a.origins, a.directions, a.ray_times = R, _ptr(origins), _ptr(directions), _ptr(ray_times)
    a.step, a.cone_angle, a.training = float(step), float(cone_angle), int(training)
    if sampler == "fixed":
        a.sampler, a.n_per_ray, a.near_plane = 0, int(n_per_ray), float(near_plane)
        cap = R * int(n_per_ray)
    elif sampler == "occupancy":
        near_planes, far_planes = _f32c(near_planes).reshape(-1), _f32c(far_planes).reshape(-1)
        b8 = binaries.detach().contiguous()
        b8 = b8.view(torch.uint8) if b8.dtype == torch.bool else b8.to(torch.uint8)
        levels, res = int(b8.shape[0]), int(b8.shape[1])
        assert b8.shape[1] == b8.shape[2] == b8.shape[3], "cubic grids only"
        ab = aabbs.detach().to(dev, _F32).reshape(levels, 6).contiguous()
        keep += [near_planes, far_planes, b8, ab]
        a.sampler = 1
        a.near_planes, a.far_planes, a.binaries, a.aabbs, a.levels, a.res = _ptr(near_planes), _ptr(far_planes), _ptr(b8), _ptr(ab), levels, res
        if capacity is None:
            diag = float((ab[:, 3:] - ab[:, :3]).norm(dim=-1).max())      # host-side: aabbs is a tiny constant buffer
            capacity = R * (int(diag / float(step)) + 2 * levels + 2)
        cap = int(capacity)
    else:
        raise ValueError(sampler)
    cap = max(cap, 1)
    a.capacity = cap
    if sampler == "occupancy" and single_traversal and cap >= R:
        scratch = torch.empty((2, cap), dtype=_F32, device=dev)      # per-ray slots of the one-traversal march
        a.march_scratch = _ptr(scratch); keep.append(scratch)
    buf = {"capacity": cap,
           "t_starts": torch.empty((cap,), dtype=_F32, device=dev), "t_ends": torch.empty((cap,), dtype=_F32, device=dev),
           "ray_indices": torch.empty((cap,), dtype=torch.int32, device=dev),
           "sigma": torch.empty((cap,), dtype=_F32, device=dev), "rgb": torch.empty((cap, 3), dtype=_F32, device=dev),
           "offsets": torch.empty((cap, 3), dtype=_F32, device=dev) if use_deformation else None,
           "weights": torch.empty((cap,), dtype=_F32, device=dev)}
    a.t_starts, a.t_ends, a.ray_indices = _ptr(buf["t_starts"]), _ptr(buf["t_ends"]), _ptr(buf["ray_indices"])
    a.sigma, a.rgb, a.offsets, a.weights = _ptr(buf["sigma"]), _ptr(buf["rgb"]), _ptr(buf["offsets"]), _ptr(buf["weights"])
    info = torch.empty((R, 2), dtype=torch.int64, device=dev)
    out = RenderResult(rgb=torch.empty((R, 3), dtype=_F32, device=dev), accumulation=torch.empty((R, 1), dtype=_F32, device=dev),
                       depth=torch.empty((R, 1), dtype=_F32, device=dev), packed_info=info)
    if use_deformation:
        out["deformation"] = torch.empty((R, 3), dtype=_F32, device=dev)
    a.packed_info, a.out_rgb, a.out_acc, a.out_depth = _ptr(info), _ptr(out["rgb"]), _ptr(out["accumulation"]), _ptr(out["depth"])
    a.out_deform = _ptr(out.get("deformation"))
    ws = torch.empty((int(lib.nsb_render_workspace_bytes(R)) + 7) // 8, dtype=torch.int64, device=dev)   # per call: results live in its header
    a.workspace = _ptr(ws)
    buf["header"] = ws          # int64 view: [barrier|depth0, depth1|status, n_total, ...]
    out["_buffers"] = buf
    out["_keep"] = keep
    out["num_samples_per_ray"] = info[:, 1]
    if R == 0:
        if want_normals:
            out["normals"] = torch.empty((0, 3), dtype=_F32, device=dev)
        return out
    opts = make_opts(window_hash, window_deform, use_deformation, True, disable_initial, soft_transition)
    frame = None
    if use_deformation:
        frame = _blended_tables(P, uniform_time, window_hash, disable_initial, soft_transition, line_gather)
    cp = P.c_params(inference=True, frame=frame)
    if mixed_linear:
        _lib.check(lib.nsb_render_forward_interp(C.byref(cp), C.byref(opts), C.byref(a), _stream()), "nsb_render_forward_interp")
    else:
        _lib.check(lib.nsb_render_forward(C.byref(cp), C.byref(opts), C.byref(a), _stream()), "nsb_render_forward")
    if want_normals:
        # the pass reads the packed samples the render left in `buf`; their count stays on the device (header n_total)
        s = _lib.Samples()
        s.n_samples, s.n_samples_dev = cap, _ptr(ws[2:3])
        s.origins, s.directions, s.ray_times = _ptr(origins), _ptr(directions), _ptr(ray_times)
        s.t_starts, s.t_ends, s.ray_indices = _ptr(buf["t_starts"]), _ptr(buf["t_ends"]), _ptr(buf["ray_indices"])
        nrm = _normals_launch(P, cp, opts, s, cap, dev, offsets=buf["offsets"], grad_scale=_world_grad_scale(P),
                              packed_info=info, weights=buf["weights"],
                              observation=use_deformation and normals_space == "observation")
        buf["normals"] = nrm["normals"]
        out["normals"] = nrm["ray_normals"]
    return out


def _flow_camera(camera, who: str):
    """(intrinsics (fx, fy, cx, cy), camera_to_world [3,4]) as host floats; a CUDA tensor is copied (one synchronisation)."""
    import math
    if not (isinstance(camera, (tuple, list)) and len(camera) == 2):
        raise ValueError(f"{who}: camera must be (intrinsics [4], camera_to_world [3,4])")
    intr = [float(v) for v in torch.as_tensor(camera[0]).detach().reshape(-1).tolist()]
    c2w = [float(v) for v in torch.as_tensor(camera[1]).detach().reshape(-1).tolist()]
    if len(intr) != 4 or len(c2w) != 12:
        raise ValueError(f"{who}: camera must be (intrinsics [4], camera_to_world [3,4])")
    if not all(math.isfinite(v) for v in intr + c2w):
        raise ValueError(f"{who}: camera values must be finite")
    if not (intr[0] > 0 and intr[1] > 0):
        raise ValueError(f"{who}: fx and fy must be > 0")
    return intr, c2w


def render_flow(P: NativeParams, result: RenderResult, origins, directions, ray_times, *, time_to: float,
                window_deform=None, camera=None, min_weight: float = FLOW_MIN_WEIGHT, max_iter: int = 20,
                tol: float = 1e-4) -> Dict[str, torch.Tensor]:
    """Scene flow and optical flow of a render_rays result from the rays' own times to `time_to` (DESIGN 4.2f), without a
    host synchronisation: nsb_flow_select picks the render's packed samples with weight >= min_weight, nsb_deform_inverse
    moves each one's canonical target c = x + offset to time_to (init x, the selected count on the device) and
    nsb_flow_composite averages the motion per ray.  origins / directions / ray_times: the ones the render was given;
    window_deform: the render's.  camera: optional (intrinsics (fx, fy, cx, cy), camera_to_world [3,4]) in the
    DeviceImageCache form, as host values (a CUDA tensor costs one synchronisation).
    Returns {"scene_flow" [R,3] world units, "flow_weight" [R,1] (the render weight the flow represents; accumulation -
    flow_weight was left out), "optical_flow" [R,2] pixels (dx right, dy down; with a camera)} plus, for tests, the
    selection ("_ray_sel" [R,2], "_sel_index", "_targets", "_init", "_n_selected") and the inverse ("_inverse"), all
    sized by the render's capacity.  Without deformation every time is the same space: zero flow, flow_weight =
    accumulation, and no flow kernel runs.  The flow follows the deformation only; occlusion at time_to is not handled."""
    import math
    _check_newton(max_iter, tol, "render_flow")
    if not (math.isfinite(float(time_to)) and 0.0 <= float(time_to) <= 1.0):
        raise ValueError(f"render_flow: time_to must be in [0, 1], got {time_to!r}")
    if not (math.isfinite(float(min_weight)) and 0.0 <= float(min_weight) < 1.0):
        raise ValueError(f"render_flow: min_weight must be finite and in [0, 1), got {min_weight!r}")
    cam = None if camera is None else _flow_camera(camera, "render_flow")
    acc = result["accumulation"]
    dev, R = acc.device, int(acc.shape[0])
    buf = result["_buffers"]
    out = {"scene_flow": torch.zeros((R, 3), dtype=_F32, device=dev)}
    if cam is not None:
        out["optical_flow"] = torch.zeros((R, 2), dtype=_F32, device=dev)
    if buf["offsets"] is None:
        out["flow_weight"] = acc.clone()
        return out
    out["flow_weight"] = torch.empty((R, 1), dtype=_F32, device=dev)
    lib = _lib.load()
    origins, directions = _f32c(origins).reshape(-1, 3), _f32c(directions).reshape(-1, 3)
    _need_cuda(origins, directions)
    assert origins.shape[0] == R and directions.shape[0] == R, (origins.shape, directions.shape, R)
    cap = int(buf["capacity"])
    sel = {"_ray_sel": torch.empty((R, 2), dtype=torch.int64, device=dev),
           "_sel_index": torch.empty((cap,), dtype=torch.int64, device=dev),
           "_targets": torch.empty((cap, 3), dtype=_F32, device=dev), "_init": torch.empty((cap, 3), dtype=_F32, device=dev),
           "_n_selected": torch.empty((1,), dtype=torch.int64, device=dev)}
    tiles = torch.empty((max((R + _lib.FLOW_TILE - 1) // _lib.FLOW_TILE, 1),), dtype=torch.int64, device=dev)
    a = _lib.FlowSelectArgs()
    a.n_rays, a.capacity, a.packed_info = R, cap, _ptr(result["packed_info"])
    a.t_starts, a.t_ends, a.weights, a.offsets = _ptr(buf["t_starts"]), _ptr(buf["t_ends"]), _ptr(buf["weights"]), _ptr(buf["offsets"])
    a.origins, a.directions, a.n_total, a.min_weight = _ptr(origins), _ptr(directions), _ptr(buf["header"][2:3]), float(min_weight)
    a.ray_sel, a.sel_index, a.targets, a.init = _ptr(sel["_ray_sel"]), _ptr(sel["_sel_index"]), _ptr(sel["_targets"]), _ptr(sel["_init"])
    a.n_selected, a.tile_sums = _ptr(sel["_n_selected"]), _ptr(tiles)
    _lib.check(lib.nsb_flow_select(C.byref(a), _stream()), "nsb_flow_select")
    inv = deform_inverse(P, sel["_targets"], uniform_time=float(time_to), init=sel["_init"], window_deform=window_deform,
                         max_iter=max_iter, tol=tol, n_samples_dev=sel["_n_selected"])
    c = _lib.FlowCompositeArgs()
    c.n_rays, c.capacity, c.ray_sel, c.sel_index = R, cap, _ptr(sel["_ray_sel"]), _ptr(sel["_sel_index"])
    c.init, c.positions, c.status, c.weights = _ptr(sel["_init"]), _ptr(inv["positions"]), _ptr(inv["status"]), _ptr(buf["weights"])
    c.scene_flow, c.flow_weight = _ptr(out["scene_flow"]), _ptr(out["flow_weight"])
    if cam is not None:
        c.intrinsics[:] = cam[0]
        c.camera_to_world[:] = cam[1]
        c.optical_flow = _ptr(out["optical_flow"])
    _lib.check(lib.nsb_flow_composite(C.byref(c), _stream()), "nsb_flow_composite")
    out.update(sel)
    out["_inverse"] = inv
    return out


MESH_SPACES = ("observation", "canonical")
MESH_SLAB_POINTS = 1 << 22          # grid points per field_forward call of the density pass
MESH_FALLBACK_DIRECTION = (0.0, 0.0, -1.0)    # colour view direction of a vertex without a normal


def mesh_grid(P: NativeParams, resolution, box=None):
    """The grid of extract_mesh: (box_min [3], h [3], (nx, ny, nz)) as Python floats already rounded to float32.
    box: [[x0, y0, z0], [x1, y1, z1]] (any nesting of 6 numbers), default the scene aabb.  An int `resolution` is the
    number of points along the longest axis with cubic voxels, h = longest extent / (resolution - 1); the other axes get
    round(extent / h) + 1 points (at least 2), so the grid ends within half a voxel of the box.  A 3-tuple (nx, ny, nz) is
    taken as given, h = extent / (n - 1) per axis."""
    import numpy as np
    b = [float(v) for v in (P.aabb_list if box is None else torch.as_tensor(box, dtype=torch.float64).reshape(-1).tolist())]
    if len(b) != 6:
        raise ValueError(f"box must hold 6 numbers (min xyz, max xyz), got {len(b)}")
    ext = [b[3 + k] - b[k] for k in range(3)]
    if min(ext) <= 0:
        raise ValueError(f"box must have a positive extent on every axis, got {ext}")
    if isinstance(resolution, int):
        if resolution < 2:
            raise ValueError("resolution must be >= 2")
        hh = max(ext) / (resolution - 1)
        dims = tuple(max(2, int(round(e / hh)) + 1) for e in ext)
        h = [hh] * 3
    else:
        dims = tuple(int(r) for r in resolution)
        if len(dims) != 3 or min(dims) < 2:
            raise ValueError(f"resolution must be an int or 3 ints, each >= 2, got {resolution!r}")
        h = [ext[k] / (dims[k] - 1) for k in range(3)]
    f32 = lambda v: float(np.float32(v))
    return [f32(b[k]) for k in range(3)], [f32(v) for v in h], dims


def density_grid(P: NativeParams, *, time: float, resolution, box=None, space: str = "observation", window_hash=None,
                 window_deform=None, binaries: Optional[torch.Tensor] = None, aabbs: Optional[torch.Tensor] = None,
                 disable_initial: bool = True, soft_transition: bool = True) -> Dict[str, object]:
    """The density pass of extract_mesh: sigma [nz, ny, nx] (x fastest) of the grid of mesh_grid at one time.
    Grid point (x, y, z) is at box_min + (x, y, z) * h, formed in float32 (product, then sum).  Density from field_forward
    at `time` (its frame table): space="observation" through the deformation, "canonical" with use_deformation=False.
    Positions are generated per z-slab of at most MESH_SLAB_POINTS points.  With binaries [levels, res, res, res] and
    aabbs [levels, 6] (an OccGridEstimator's), sigma is 0 at points whose occupancy cell is empty, as the marcher skips
    them: the first level whose box contains the point decides, points outside every level are empty.  The outermost
    layer of grid points is set to 0, so every isosurface at a level >= 0 is closed.
    Returns {"sigma", "box_min", "h"}."""
    if space not in MESH_SPACES:
        raise ValueError(f"space must be one of {MESH_SPACES}, got {space!r}")
    if (binaries is None) != (aabbs is None):
        raise ValueError("binaries and aabbs go together")
    dev = P.tables.device
    box_min, h, (nx, ny, nz) = mesh_grid(P, resolution, box)
    if nx * ny * nz >= (1 << 31):
        raise ValueError(f"the grid {nx} x {ny} x {nz} has 2^31 points or more")
    sigma = torch.empty((nz, ny, nx), dtype=_F32, device=dev)
    axis = [torch.arange(n, device=dev, dtype=_F32) * h[k] + box_min[k] for k, n in enumerate((nx, ny, nz))]
    occ = None
    if binaries is not None:
        _need_cuda(binaries, aabbs)
        occ = binaries.detach().to(torch.bool)
        L, res = int(occ.shape[0]), int(occ.shape[1])
        assert occ.shape[1:] == (res, res, res), "cubic occupancy grids only"
        occ_ab = aabbs.detach().to(dev, _F32).reshape(L, 6)
    slab = max(1, MESH_SLAB_POINTS // (nx * ny))
    obs = space == "observation"
    for z0 in range(0, nz, slab):
        z1 = min(nz, z0 + slab)
        Z, Y, X = torch.meshgrid(axis[2][z0:z1], axis[1], axis[0], indexing="ij")
        pos = torch.stack([X, Y, Z], -1).reshape(-1, 3)
        n = pos.shape[0]
        s = field_forward(P, window_hash=window_hash, window_deform=window_deform, use_deformation=obs, positions=pos,
                          sample_times=torch.full((n,), float(time), dtype=_F32, device=dev), uniform_time=float(time),
                          want=("sigma",), disable_initial=disable_initial, soft_transition=soft_transition)["sigma"]
        if occ is not None:
            keep = torch.zeros((n,), dtype=torch.bool, device=dev)
            seen = torch.zeros((n,), dtype=torch.bool, device=dev)
            for l in range(L):        # the march's cell of a position: int(((p - aabb_min) / extent) * res)
                lo, hi = occ_ab[l, :3], occ_ab[l, 3:]
                u = (pos - lo) / (hi - lo)
                inl = ((u >= 0) & (u < 1)).all(-1)
                c = (u * res).long().clamp_(0, res - 1)
                keep |= inl & ~seen & occ[l][c[:, 0], c[:, 1], c[:, 2]]
                seen |= inl
            s = torch.where(keep, s, torch.zeros_like(s))
        sigma[z0:z1].view(-1).copy_(s)
    for v in (sigma[0], sigma[-1], sigma[:, 0], sigma[:, -1], sigma[:, :, 0], sigma[:, :, -1]):
        v.zero_()
    return {"sigma": sigma, "box_min": box_min, "h": h}


def marching_tetrahedra(sigma: torch.Tensor, level: float, box_min, h) -> Dict[str, torch.Tensor]:
    """Isosurface {sigma = level} of a grid sigma [nz, ny, nx] (x fastest), grid point (x, y, z) at box_min + (x, y, z) * h
    (nsb_mesh_count / nsb_mesh_emit): marching tetrahedra on the Kuhn split, inside = sigma > level.  Returns
    {"vertices" [V,3] float32, "faces" [F,3] int32}: one vertex per crossing grid edge, ids in (grid point, edge slot)
    order, faces in (cell, tetrahedron, triangle) order, counter-clockwise seen from outside (DESIGN 4.2d).  The same bits
    on every run.  Reads the two totals back with ONE host synchronisation to allocate exact-size outputs: this is an
    export, not a render path."""
    _need_cuda(sigma)
    if sigma.dim() != 3:
        raise ValueError(f"sigma must be [nz, ny, nx], got {tuple(sigma.shape)}")
    sg = _f32c(sigma)
    nz, ny, nx = (int(v) for v in sg.shape)
    dev = sg.device
    a = _lib.MeshArgs()
    a.sigma, a.nx, a.ny, a.nz, a.level = _ptr(sg), nx, ny, nz, float(level)
    for k in range(3):
        a.box_min[k], a.h[k] = float(box_min[k]), float(h[k])
    lib = _lib.load()
    n = nx * ny * nz
    tiles = (n + _lib.MESH_TILE - 1) // _lib.MESH_TILE
    point_mask = torch.empty((max(n, 1),), dtype=torch.uint8, device=dev)
    vertex_base = torch.empty((max(n, 1),), dtype=torch.int32, device=dev)
    tile_sums = torch.empty((2 * tiles + 2,), dtype=torch.int64, device=dev)
    a.point_mask, a.vertex_base, a.tile_sums = _ptr(point_mask), _ptr(vertex_base), _ptr(tile_sums)
    _lib.check(lib.nsb_mesh_count(C.byref(a), _stream()), "nsb_mesh_count")
    V, F = tile_sums[2 * tiles:].tolist()           # the one host synchronisation: exact-size outputs
    if V >= (1 << 31) or F >= (1 << 31):
        raise RuntimeError(f"marching_tetrahedra: {V} vertices / {F} faces do not fit int32 ids; use a coarser grid")
    out = {"vertices": torch.empty((V, 3), dtype=_F32, device=dev), "faces": torch.empty((F, 3), dtype=torch.int32, device=dev)}
    a.n_vertices, a.n_faces = V, F
    a.vertices, a.faces = _ptr(out["vertices"]), _ptr(out["faces"])
    _lib.check(lib.nsb_mesh_emit(C.byref(a), _stream()), "nsb_mesh_emit")
    return out


def extract_mesh(P: NativeParams, *, time: float, level: float, resolution, box=None, space: str = "observation",
                 window_hash=None, window_deform=None, binaries: Optional[torch.Tensor] = None,
                 aabbs: Optional[torch.Tensor] = None, normals: bool = True, colours: bool = True,
                 disable_initial: bool = True, soft_transition: bool = True) -> Dict[str, torch.Tensor]:
    """Surface mesh of the density field at one time: density_grid, then marching_tetrahedra at `level` (>= 0), then
    per-vertex normals and colours.  space="observation" is the observed (deformed) head of that frame, "canonical" the
    surface the field stores.  Returns {"vertices" [V,3] float32 world, "faces" [F,3] int32, "normals" [V,3],
    "colours" [V,3]} (normals / colours only when asked for).
    normals: field_normals at the vertices in the same space, world space; zero where the warped position leaves the box.
    colours: field_forward RGB seen head-on, view direction -normal (MESH_FALLBACK_DIRECTION where the normal is zero).
    One host synchronisation (the mesh size); not differentiable."""
    import math
    if not math.isfinite(float(level)) or float(level) < 0:
        raise ValueError(f"level must be finite and >= 0 (sigma is non-negative), got {level}")
    g = density_grid(P, time=time, resolution=resolution, box=box, space=space, window_hash=window_hash,
                     window_deform=window_deform, binaries=binaries, aabbs=aabbs, disable_initial=disable_initial,
                     soft_transition=soft_transition)
    out = marching_tetrahedra(g["sigma"], level, g["box_min"], g["h"])
    del g
    out.update(vertex_attributes(P, out["vertices"], time=time, space=space, normals=normals, colours=colours,
                                 window_hash=window_hash, window_deform=window_deform, disable_initial=disable_initial,
                                 soft_transition=soft_transition))
    return out


def vertex_attributes(P: NativeParams, vertices: torch.Tensor, *, time: float, space: str = "observation",
                      normals: bool = True, colours: bool = True, sigma: bool = False, window_hash=None, window_deform=None,
                      disable_initial: bool = True, soft_transition: bool = True) -> Dict[str, torch.Tensor]:
    """The per-vertex attributes of extract_mesh at world `vertices` [V,3] and one time: "normals" (field_normals in
    `space`, world space, zero where the warped position leaves the box), "colours" (field_forward RGB seen head-on, view
    direction -normal, MESH_FALLBACK_DIRECTION where the normal is zero) and "sigma" (the density there), each when asked
    for."""
    out: Dict[str, torch.Tensor] = {}
    if not (normals or colours or sigma):
        return out
    v = vertices
    V, dev = int(v.shape[0]), v.device
    obs = space == "observation"
    kw = dict(window_hash=window_hash, positions=v, sample_times=torch.full((V,), float(time), dtype=_F32, device=dev),
              uniform_time=float(time), disable_initial=disable_initial, soft_transition=soft_transition)
    if normals or colours:
        off = field_forward(P, window_deform=window_deform, want=("offsets",), **kw)["offsets"] if obs else None
        nrm = field_normals(P, offsets=off, world_space=True, space=space, window_deform=window_deform, **kw)["normals"]
        if normals:
            out["normals"] = nrm
    if colours:
        fb = torch.tensor(MESH_FALLBACK_DIRECTION, dtype=_F32, device=dev)
        dirs = torch.where((nrm == 0).all(-1, keepdim=True), fb, -nrm)
        out["colours"] = field_forward(P, window_deform=window_deform, use_deformation=obs, sample_directions=dirs,
                                       want=("rgb",), **kw)["rgb"]
    if sigma:
        out["sigma"] = field_forward(P, window_deform=window_deform, use_deformation=obs, want=("sigma",), **kw)["sigma"]
    return out


def extract_mesh_sequence(P: NativeParams, *, times: Sequence[float], reference_time: float, level: float, resolution,
                          box=None, space: str = "observation", window_hash=None, window_deform=None,
                          binaries: Optional[torch.Tensor] = None, aabbs: Optional[torch.Tensor] = None,
                          normals: bool = True, colours: bool = True, disable_initial: bool = True,
                          soft_transition: bool = True, max_iter: int = 20, tol: float = 1e-4) -> Dict[str, object]:
    """A mesh sequence with one connectivity: extract_mesh's mesh of the frame at `reference_time` (no attributes), its
    vertices tracked to every time in `times` (track_points; space="observation"), and per frame the vertex attributes of
    extract_mesh at the tracked vertices plus sigma there.  space="canonical" (or a field without deformation, when the
    caller passes it) keeps the reference mesh's vertices in every frame.  Returns {"faces" [F,3], "vertices" [K,V,3],
    "converged" [K,V], "residual" [K,V], "sigma" [K,V], "normals" / "colours" [K,V,3] (when asked for)}."""
    _check_newton(max_iter, tol, "extract_mesh_sequence")
    ref = extract_mesh(P, time=reference_time, level=level, resolution=resolution, box=box, space=space,
                       window_hash=window_hash, window_deform=window_deform, binaries=binaries, aabbs=aabbs, normals=False,
                       colours=False, disable_initial=disable_initial, soft_transition=soft_transition)
    v0 = ref["vertices"]
    V, dev = int(v0.shape[0]), v0.device
    times = [float(t) for t in times]
    if space == "observation" and V > 0:
        tr = track_points(P, v0, time_from=float(reference_time), times_to=times, window_deform=window_deform,
                          max_iter=max_iter, tol=tol)
    else:
        K = len(times)
        tr = {"positions": v0.unsqueeze(0).expand(K, V, 3).contiguous(), "residual": torch.zeros((K, V), dtype=_F32, device=dev),
              "converged": torch.ones((K, V), dtype=torch.bool, device=dev)}
    out: Dict[str, object] = {"faces": ref["faces"], "vertices": tr["positions"], "converged": tr["converged"],
                              "residual": tr["residual"]}
    per = [vertex_attributes(P, tr["positions"][i], time=t, space=space, normals=normals, colours=colours, sigma=True,
                             window_hash=window_hash, window_deform=window_deform, disable_initial=disable_initial,
                             soft_transition=soft_transition) for i, t in enumerate(times)]
    for k in ("sigma", "normals", "colours"):
        if per and k in per[0]:
            out[k] = torch.stack([p[k] for p in per])
    return out


def render_packed(P: NativeParams, origins, directions, ray_times, t_starts, t_ends, ray_indices, packed_info, *,
                  window_hash=None, window_deform=None, use_deformation=True, training=False,
                  disable_initial=True, soft_transition=True, sample_blend_codes=None,
                  sample_warp_codes=None) -> Dict[str, torch.Tensor]:
    """NeRSembleNGPModel.get_outputs after the sampler (nersemble_instant_ngp.py:297-364).  sample_blend_codes [n,32] /
    sample_warp_codes [n,128]: per-sample codes instead of the rows of the ray times (field_forward)."""
    f = field_forward(P, window_hash=window_hash, window_deform=window_deform, use_deformation=use_deformation,
                      origins=origins, directions=directions, ray_times=ray_times, t_starts=t_starts, t_ends=t_ends,
                      ray_indices=ray_indices, want=("sigma", "rgb", "offsets"), sample_blend_codes=sample_blend_codes,
                      sample_warp_codes=sample_warp_codes if use_deformation else None,
                      disable_initial=disable_initial, soft_transition=soft_transition)
    c = composite(packed_info, t_starts, t_ends, f["sigma"], f["rgb"], f["offsets"] if use_deformation else None,
                  training=training)
    c["num_samples_per_ray"] = packed_info[:, 1]
    c["offsets"] = f["offsets"]
    c["density"] = f["sigma"][:, None]
    c["rgb_samples"] = f["rgb"]
    return c
