"""The training backward at batch scale: 2^19-entry tables, T = 24, ~150 k ray-ordered samples, so that every CTA of
field_mlp_bwd_kernel / deform_bwd_kernel runs several tiles, every hash warp a run of several samples (timestep changes
and ray boundaries inside a run, merged runs in the saved-corner kernel) and hash_expand_kernel / table_step_kernel many
grid-stride passes.  test_gpu_backward.py pins the per-tile mathematics to autograd at small size; here the reduction
structure is checked, stage by stage on the inputs the previous stage produced:

  * per-sample outputs are bit-identical between one launch and launches on chunks of at most 64 tiles (one tile per
    CTA, at most one sample per hash warp: the regime the small tests cover);
  * reductions of the one launch equal the float64 sum of the chunked launches, within float32 reduction noise;
  * the hash-grid gradients equal the float64 references of backward_scale_oracle within rigorous float32 bounds.

Every bound is derived next to its assertion, and each bounded check is shown, on the reference side, to reject a
realistic bug by at least 10x."""
import math

import pytest
import torch

from backward_scale_oracle import (U32, code_grad_from_G, cw16, dense_table_grad, hash_scatter_ref, per_sample_terms)
from conftest import native_from_oracle, oracle_params
from oracle.tp.tcnn_cpu import Precision

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
FULL = dict(seed=19980801, n_timesteps=24, log2_hashmap_size=19, table_scale=0.5, time_std_scale=100.0,
            deform_last_scale=1e-3)
T48 = dict(FULL, n_timesteps=48, log2_hashmap_size=14)
R_RAYS, PER_RAY = 1210, 127            # 153 670 samples: 1 201 tiles, the last one ragged (70 rows)
SMS = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 0
# chunked launches: at most 64 tiles, and few enough for one tile per CTA and one sample per hash warp (64 SMS warps)
CHUNK_TILES = min(64, SMS // 2) if SMS else 64
W_HASH, W_DEFORM = 20.25, 5.5          # w_hash >= 2: the blend-weight fold has a zero bias (see backward_scale_oracle.cw16)
LS_FIELD, LS_DEFORM = 128.0, 64.0
N = R_RAYS * PER_RAY
N_TILES = (N + 127) // 128
if SMS:
    # what the batch has to reach on this device, or the paths this file exists for are not covered
    assert N_TILES >= 4 * SMS, "fewer than 4 tiles per CTA"
    assert N >= 4 * 64 * SMS, "fewer than 4 samples per hash warp"
    assert CHUNK_TILES <= SMS and CHUNK_TILES * 128 <= 64 * SMS, "a chunk must give one tile per CTA, one sample per hash warp"


@pytest.fixture(autouse=True)
def _mode():
    Precision.mode = "kernel"; Precision.autocast = False
    yield
    Precision.mode = "reference"
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True, scope="module")
def _free_module_caches():
    yield
    _BATCH.clear(); _MODES.clear()
    torch.cuda.empty_cache()


def _chunks(n):
    step = CHUNK_TILES * 128
    return [(a, min(n, a + step)) for a in range(0, n, step)]


def _rays(T, seed, time_of_ray=None):
    from nersemble_b200 import ops
    from oracle.gen_golden import ring_rays
    P = oracle_params(T if isinstance(T, dict) else FULL)
    o, d, times, _ = ring_rays(R_RAYS, seed)
    nt = P.n_timesteps
    if time_of_ray is None:
        times[:nt, 0] = torch.arange(nt) / (nt - 1)        # every timestep occurs; the rest stay unsorted
    else:
        times[:, 0] = time_of_ray(nt)
    o[7] = torch.tensor([50.0, 50.0, 50.0]); d[7] = torch.tensor([0.0, 1.0, 0.0])          # rays that miss the box
    o[400] = torch.tensor([-50.0, 0.0, 0.0]); d[400] = torch.tensor([0.0, 0.0, 1.0])
    o, d, times = o.to(DEV), d.to(DEV), times.to(DEV)
    ts, te, ri, _ = ops.march_fixed(o, d, P.aabb, PER_RAY, 0.011, 0.2)
    # timestep of every sample, as the kernels round it: __float2int_rn(t * (T - 1))
    tsi = (times[:, 0][ri.long()] * float(nt - 1)).round().clamp(0, nt - 1).long()
    return P, dict(origins=o, directions=d, ray_times=times, t_starts=ts, t_ends=te, ray_indices=ri), tsi


def _rows_kw(kw, a, b):
    return dict(origins=kw["origins"], directions=kw["directions"], ray_times=kw["ray_times"],
                t_starts=kw["t_starts"][a:b], t_ends=kw["t_ends"][a:b], ray_indices=kw["ray_indices"][a:b])


_BATCH = {}


def _batch(knobs=None, seed=17, time_of_ray=None, key="full"):
    """Forward of the batch (saved tensors of the training forward) and the upstream gradients, cached per key."""
    from nersemble_b200 import ops
    if key not in _BATCH:
        _BATCH.clear(); torch.cuda.empty_cache()
        P, kw, tsi = _rays(knobs or FULL, seed, time_of_ray)
        NP = native_from_oracle(P, DEV)
        saved = ops.field_forward(NP, window_hash=W_HASH, window_deform=W_DEFORM, use_deformation=True,
                                  want=("sigma", "rgb", "feat", "xs", "corner_vals", "deform_acts"), **kw)
        g = torch.Generator(device=DEV).manual_seed(seed)
        up = dict(d_sigma=torch.randn((N,), generator=g, device=DEV) * 0.1, d_rgb=torch.randn((N, 3), generator=g, device=DEV),
                  d_xs=torch.randn((N, 3), generator=g, device=DEV))
        _BATCH[key] = (P, NP, kw, tsi, saved, up)
    return _BATCH[key]


def _saved_rows(saved, a, b):
    return {k: saved[k][a:b] for k in ("sigma", "rgb", "feat", "xs", "corner_vals")}


def _field_bwd(NP, saved, up, kw, a, b, mode, **extra):
    from nersemble_b200 import ops
    cv = mode in ("saved_corners", "deferred")
    s = _saved_rows(saved, a, b)
    if not cv:
        s.pop("corner_vals")
    return ops.field_backward(NP, s, up["d_sigma"][a:b], up["d_rgb"][a:b], window_hash=W_HASH, loss_scale=LS_FIELD,
                              want_dx=True, rank1=mode != "direct", defer_tables=mode == "deferred",
                              **_rows_kw(kw, a, b), **extra)


def _scale_bias():
    from nersemble_b200 import packing
    return packing.blend_fold(W_HASH, 32, True, True)


def _assert_within(got, want, bound, what):
    """max |got - want| / bound <= 1 (elements with a zero bound must match exactly)."""
    err = (got.double() - want.double()).abs()
    bad = err > bound
    assert not bad.any(), (f"{what}: {int(bad.sum())} elements over the bound, worst err {err.max().item():.3e}, "
                           f"ratio {(err / bound.clamp_min(1e-300)).max().item():.3e}")


def _rejects(delta, bound, what):
    """Negative control: the planted error `delta` exceeds the bound 10x somewhere."""
    r = (delta.abs() / bound.clamp_min(1e-300)).max().item()
    assert r >= 10.0, f"negative control '{what}': the bound only sees {r:.2f}x of the planted error"


# ---------------------------------------------------------------------------------------------------------------------
# hash-grid gradients (c) + chunked launches (a, b) + the MLP weight gradients (b)
# ---------------------------------------------------------------------------------------------------------------------
_MODES = {}         # per scatter mode: outputs and bounds, to check the four modes against each other


def _hash_ref(levels, xs, d_feat, sample_slot, n_slots):
    G, A, K, touched = hash_scatter_ref(levels, xs, d_feat, sample_slot, n_slots)
    return dict(G=G, A=A, K=K, touched=touched)


def _any_order(terms):
    """sum_k |S_k| over the partial sums of the terms (dim 0) added in the worst order: |S_k| <= the sum of the k
    largest |terms|, and |S_k| = |total - rest| <= |total| + the sum of the n - k largest.  A float32 sum whose first
    add goes into zero rounds by at most u |S_k| per later add, so u times this bounds it in any order."""
    a = terms.abs().sort(0, descending=True).values
    top = torch.cumsum(a, 0)                                              # top[k - 1]: the k largest
    rest = torch.cat([top.flip(0)[1:], torch.zeros_like(top[:1])], 0)     # rest[k - 1]: the n - k largest
    return torch.minimum(top, terms.sum(0).abs() + rest).sum(0)


def _check_dense_tables(got, ref, cw_slots, what, lines_step=1 << 19):
    """Dense [E, 32, 2] table gradient against the reference, per entry:
        |got - ref| <= 2 u (K_e + 2) A_e.
    Direct scatter: each of the K_e terms is fl(fl(w * dfeat) * cw) (two roundings) and is added by a float32 atomic
    in some order: |err| <= (K_e + 1) u A_e to first order (A_e = sum of |terms|).  Rank-1 path: per slot K_s terms
    fl(w * dfeat) summed in float32 ((K_s) u A_s), then the expansion's fma chain over the touched slots (<= K_e more
    roundings) -- together <= (2 K_e) u A_e.  The factor 2 (K_e + 2) covers both plus second-order terms; K_e is small
    for all but the coarse levels, so the bound is tight where a lost contribution would hide.  Untouched lines must be
    exactly zero and the touched line sets identical."""
    G, A, K = ref["G"], ref["A"], ref["K"]
    E = G.shape[1]
    got_touched = torch.zeros(E, dtype=torch.bool, device=DEV)
    for a in range(0, E, lines_step):
        lines = torch.arange(a, min(E, a + lines_step), device=DEV)
        r, ab, k = dense_table_grad(G, A, K, cw_slots, lines)
        bound = 2 * U32 * (k[:, None, None] + 2) * ab
        _assert_within(got[a:a + lines.numel()], r, bound, what)
        got_touched[a:a + lines.numel()] = (got[a:a + lines.numel()] != 0).flatten(1).any(1)
    # a line is touched when some slot has a non-zero contribution and a non-zero blend weight multiplies it
    nz_member = (cw_slots != 0).any(1)                                          # slots whose weights are not all zero
    want_touched = (ref["touched"] & nz_member[:, None]).any(0)
    assert torch.equal(got_touched, want_touched), f"{what}: touched lines differ ({int((got_touched ^ want_touched).sum())})"


def _segments(tsi, n_launch, n_t):
    """(warp, timestep) runs of hash_bwd_kernel: warp w takes samples [w per, (w + 1) per), per = ceil(n / (64 SMS)),
    and flushes its code sum whenever the timestep changes.  Returns (segment id per sample, timestep per segment, per)."""
    n = tsi.numel()
    per = (n_launch + 64 * SMS - 1) // (64 * SMS)
    key = (torch.arange(n, device=DEV) // per) * n_t + tsi
    start = torch.ones(n, dtype=torch.bool, device=DEV); start[1:] = key[1:] != key[:-1]
    return torch.cumsum(start.long(), 0) - 1, tsi[start], per


def _next_occurring(tsi, n_t):
    """t -> the next timestep that occurs in the batch (cyclic)."""
    uniq = torch.unique(tsi)
    nxt = torch.full((n_t,), -1, dtype=torch.long, device=DEV)
    nxt[uniq] = torch.roll(uniq, -1)
    return nxt


def _run_control(code_s, tsi, bound, n_t):
    """Negative control: one hash warp's run credited to the neighbouring timestep (the next one that occurs) moves
    the run's code sum from t to there.  The control takes the run that moves the gradient most relative to the bound
    (a bug that mis-credits runs mis-credits that one too).  Returns the run's (first row, timestep)."""
    seg, seg_t, per = _segments(tsi, tsi.numel(), n_t)
    nxt = _next_occurring(tsi, n_t)
    run = torch.zeros((seg_t.numel(), 32), dtype=torch.float64, device=DEV).index_add_(0, seg, code_s)
    ratio = (run.abs() / bound[seg_t].clamp_min(1e-300)).amax(1)
    r0 = int(ratio.argmax())
    t0, t1 = int(seg_t[r0]), int(nxt[seg_t[r0]])
    delta = torch.zeros_like(bound)
    delta[t0] -= run[r0]; delta[t1] += run[r0]
    _rejects(delta, bound, "a warp's run credited to the neighbouring timestep")
    return (seg == r0).nonzero()[:, 0], t0, t1


def _code_bound_direct(code_abs_t, c_abs_t, tsi, n_launch, n_t):
    """hash_bwd_kernel's code gradient (direct scatter).  Per sample and member: a 33-deep float32 chain (g = w * dfeat,
    then 2 fmas per level) + 3 shuffle adds + the x cw_scale product: <= 40 u of the sample's abs-sum (code_abs).  Then
    the warp adds its run's samples (<= per terms) and flushes with one atomic per (run, timestep) segment: W_t atomics
    per timestep, summed in any order.  |err_t| <= u [40 A_t + (per + W_t + 1) C_t], C_t = sum over samples of the
    per-sample |code| (the outer sums add per-sample values, not their terms)."""
    _, seg_t, per = _segments(tsi, n_launch, n_t)
    W_t = torch.bincount(seg_t, minlength=n_t).double()
    return U32 * (40 * code_abs_t + (per + W_t[:, None] + 1) * c_abs_t)


def _code_bound_rank1_order(ref, V, sc, slot_ts, n_t):
    """hash_expand_kernel's code gradient, bounded along the order in which it sums.  Warp w of the W = 24 SMS warps
    (SMS * 6 blocks of 4) takes the 32-line blocks blk = w, w + W, ... and, per touched line in ascending order, adds
    V[e, m, 0] G[e, 0] + V[e, m, 1] G[e, 1] to its running sum with two fmas; each warp then adds its sum P_w with one
    atomic, and the result is multiplied by cw_scale.  With the float32 G carrying <= (K + 1) u A per (entry, f):
      |err| <= |cw_scale| u [ sum_{e,f} |V| (K + 1) A                 (G as the rank-1 scatter left it)
                              + 2 sum_w sum_{e in w} (|prefix_e| + |term_e|)   (each fma rounds at most its running sum)
                              + _any_order(P_w) + sum_w |P_w| ]     (the atomics of P_w cw_scale, in any order)
                 + u |code|                                             (slack for second-order terms)
    evaluated on the float64 G (the difference is second order).  Lines nobody touched add zero terms here, which
    only enlarges the prefix sum."""
    G, A, K = ref["G"], ref["A"], ref["K"]
    S, E, _ = G.shape
    W = SMS * 6 * 4
    span = W * 32                                        # one grid-stride round: 32 lines of every warp
    run = torch.zeros((S, W, 32), dtype=torch.float64, device=DEV)       # running sum of each (slot, warp, member)
    inner = torch.zeros((S, 32), dtype=torch.float64, device=DEV)
    chain = torch.zeros_like(inner)
    for a in range(0, E, span):
        b = min(E, a + span)
        Vd = V[a:b].double()
        inner += torch.einsum("emf,sef->sm", Vd.abs(), (K[:, a:b, None].double() + 1) * A[:, a:b])
        term = torch.zeros((S, span, 32), dtype=torch.float64, device=DEV)
        term[:, :b - a] = torch.einsum("emf,sef->sem", Vd, G[:, a:b])
        term = term.view(S, W, 32, 32)                   # [slot, warp, its 32 lines of this round, member]
        pre = run[:, :, None, :] + torch.cumsum(term, 2)
        chain += 2 * (pre.abs().sum((1, 2)) + term.abs().sum((1, 2)))
        run = pre[:, :, -1]
    sc64 = torch.as_tensor(sc, dtype=torch.float32, device=DEV).double().abs()
    out = torch.zeros((n_t, 32), dtype=torch.float64, device=DEV)
    atom = _any_order(run.transpose(0, 1)) + run.abs().sum(1)
    out[slot_ts] = sc64 * U32 * (inner + chain + atom) + U32 * (sc64 * run.sum(1)).abs()
    return out


def _chunk_code_bounds(mode, levels, saved, d_feat, tsi, code_abs_s, code_s, V, sc, slot_map, slot_ts, n_slots, n_t):
    """Bounds of each chunked launch's code gradient, from the chunk's own structure: the direct scatter's per-chunk
    segments (one sample per warp), or the order of hash_expand_kernel over the chunk's own G."""
    out = []
    for a, b in _chunks(tsi.numel()):
        t = tsi[a:b]
        if mode == "direct":
            ca = torch.zeros((n_t, 32), dtype=torch.float64, device=DEV).index_add_(0, t, code_abs_s[a:b])
            cc = torch.zeros_like(ca).index_add_(0, t, code_s[a:b].abs())
            out.append(_code_bound_direct(ca, cc, t, b - a, n_t))
        else:
            r = _hash_ref(levels, saved["xs"][a:b], d_feat[a:b], slot_map[t], n_slots)
            out.append(_code_bound_rank1_order(r, V, sc, slot_ts, n_t))
            del r
    return torch.stack(out)


def _check_codes(one_codes, ch_codes, code_t, bound_one, bound_ch, what):
    """One launch and chunk sum against float64, the two against each other, and the chunk-left-out control."""
    _assert_within(one_codes, code_t, bound_one, f"{what}: d_blend_codes")
    _assert_within(ch_codes.sum(0), code_t, bound_ch.sum(0), f"{what}: d_blend_codes of the chunks")
    _assert_within(one_codes, ch_codes.sum(0), bound_one + bound_ch.sum(0), f"{what}: d_blend_codes one vs chunks")
    for k in range(ch_codes.shape[0]):        # one chunk left out of the chunk sum
        _rejects(ch_codes[k], bound_one + bound_ch.sum(0), f"{what}: d_blend_codes without chunk {k}")


def _table_run_control(levels, saved, d_feat, rows, ref, cw_slots, s0, s1):
    """Negative control on the dense table gradient: the rows of one hash warp's run credited to timestep t1 instead
    of t0 (slots s1, s0) change the lines they touch by (cw[s1] - cw[s0]) x their G."""
    Gr, _, _, touched = hash_scatter_ref(levels, saved["xs"][rows], d_feat[rows], torch.zeros_like(rows), 1)
    lines = touched[0].nonzero()[:, 0]
    r, ab, k = dense_table_grad(ref["G"], ref["A"], ref["K"], cw_slots, lines)
    delta = (cw_slots[s1] - cw_slots[s0])[None, :, None] * Gr[0, lines][:, None, :]
    _rejects(delta, 2 * U32 * (k[:, None, None] + 2) * ab, "a warp's run credited to the neighbouring timestep (tables)")
    return Gr[0], touched[0]


@pytest.mark.parametrize("mode", ["direct", "rank1", "saved_corners", "deferred"])
def test_field_backward_at_batch_scale(mode):
    from nersemble_b200 import ops
    from oracle.tp.tcnn_cpu import hashgrid_indices_weights
    P, NP, kw, tsi, saved, up = _batch()
    E, T = P.levels.total_entries, P.n_timesteps
    sc, bi = _scale_bias()
    V = NP.tables
    one = _field_bwd(NP, saved, up, kw, 0, N, mode)
    # the chunks' table gradients are folded into float64 sums as they come (19 dense gradients would be 30 GB)
    ch_dense = torch.zeros((E, 32, 2), dtype=torch.float64, device=DEV)
    ch_g1 = torch.zeros((T, E, 2), dtype=torch.float64, device=DEV) if mode == "deferred" else None
    chunks = []
    for a, b in _chunks(N):
        c = _field_bwd(NP, saved, up, kw, a, b, mode)
        if mode == "deferred":
            ch_g1 += c["pending"]["g_rank1"]
            ch_dense += ops.rank1_expand(c.pop("pending"), E)
        else:
            ch_dense += c.pop("d_tables")
        chunks.append(c)

    # (a) per-sample outputs: each row's arithmetic is independent of the CTA / warp that handles it
    assert torch.equal(torch.cat([c["d_feat"] for c in chunks]), one["d_feat"])
    assert torch.equal(torch.cat([c["d_xs"] for c in chunks]), one["d_xs"])
    d_feat = one["d_feat"]

    # (b) the MLP weight gradients: per-tile launches give each tile's exact contribution t (one CTA, one tile: the
    # accumulator starts at zero, x 1/loss_scale is exact, one atomic into zero).  The one launch sums <= ceil(tiles /
    # SMS) tiles per CTA in shared memory, then SMS atomics; a chunk CHUNK_TILES atomics:
    # |err| <= u (tiles_per_cta + SMS + CHUNK_TILES) M with M = sum |t| over tiles (+ 8: the float64 sum, second order)
    if mode == "direct":
        # (only the weight gradients are kept: each launch's per-sample buffers are 65 536-row allocations)
        tiles = [{k: v for k, v in ops.field_backward(
                     NP, _saved_rows(saved, a, min(N, a + 128)), up["d_sigma"][a:a + 128], up["d_rgb"][a:a + 128],
                     window_hash=W_HASH, loss_scale=LS_FIELD, want_tables=False, want_codes=False,
                     **_rows_kw(kw, a, min(N, a + 128))).items() if k in ("d_base_w", "d_head_w")}
                 for a in range(0, N, 128)]
        for name in ("d_base_w", "d_head_w"):
            t = torch.stack([x[name] for x in tiles]).double()
            exact, M = t.sum(0), t.abs().sum(0)
            bound = U32 * (math.ceil(N_TILES / SMS) + SMS + CHUNK_TILES + 8) * M
            ch = torch.stack([c[name] for c in chunks]).double()
            _assert_within(one[name], exact, bound, f"{name}: one launch vs the sum of its tiles")
            _assert_within(ch.sum(0), exact, bound, f"{name}: chunked launches vs the sum of the tiles")
            _assert_within(one[name], ch.sum(0), 2 * bound, f"{name}: one launch vs chunked launches")
            for k in range(ch.shape[0]):       # what "one tile per CTA dropped" looks like, for every chunk
                _rejects(ch[k], 2 * bound, f"{name} without chunk {k}")
        del tiles

    # (c) hash-grid gradients against float64
    cw_t = cw16(NP.blend_codes, sc, bi)                                   # [T, 32]
    cv = saved["corner_vals"] if mode in ("saved_corners", "deferred") else None
    code_s, code_abs_s, dxs_ref, dxs_abs = per_sample_terms(P.levels, saved["xs"], d_feat, V, cw_t[tsi], sc, corner_vals=cv)
    # d_xs: table path a chain of <= 33 roundings per term (8-member fma blend, t = scale (df . pb) 3, w_y w_z 1,
    # 16-level fma chain, 5 shuffle adds); saved corners <= 13 (t 3, 1, 4-deep chain, 5 shuffles): 40 / 16 u of the
    # per-sample abs-sum of the expanded terms
    n_dx = 16 if cv is not None else 40
    dx_bound = n_dx * U32 * dxs_abs
    _assert_within(one["d_xs"], dxs_ref, dx_bound, f"{mode}: d_xs")
    # negative control: one sample's finest-level term of d_xs dropped
    s0 = int((d_feat[:, 30:].abs().sum(1) * saved["xs"][:, 3]).argmax())
    df15 = torch.zeros_like(d_feat[s0:s0 + 1]); df15[:, 30:] = d_feat[s0:s0 + 1, 30:]
    _, _, dx15, _ = per_sample_terms(P.levels, saved["xs"][s0:s0 + 1], df15, V, cw_t[tsi[s0:s0 + 1]], sc,
                                     corner_vals=None if cv is None else cv[s0:s0 + 1])
    _rejects(dx15, dx_bound[s0:s0 + 1], "one sample's finest-level d_xs term dropped")

    code_t = torch.zeros((T, 32), dtype=torch.float64, device=DEV).index_add_(0, tsi, code_s)
    code_abs_t = torch.zeros_like(code_t).index_add_(0, tsi, code_abs_s)
    c_abs_t = torch.zeros_like(code_t).index_add_(0, tsi, code_s.abs())
    slot = torch.arange(T, device=DEV)
    bound_ch = _chunk_code_bounds(mode, P.levels, saved, d_feat, tsi, code_abs_s, code_s, V, sc, slot, slot, T, T)
    ref = _hash_ref(P.levels, saved["xs"], d_feat, tsi, T)
    if mode == "direct":
        assert (code_grad_from_G(ref["G"], V, sc) - code_t).abs().max() <= 1e-9 * code_abs_t.max()   # the two float64 routes
        bound_one = _code_bound_direct(code_abs_t, c_abs_t, tsi, N, T)
    else:
        bound_one = _code_bound_rank1_order(ref, V, sc, slot, T)
    ch_codes = torch.stack([c["d_blend_codes"] for c in chunks]).double()
    _check_codes(one["d_blend_codes"], ch_codes, code_t, bound_one, bound_ch, mode)
    # negative control for every mode: one hash warp's run credited to the neighbouring timestep.  In the rank-1 modes
    # the run lands in the wrong slot of G and reaches the code gradient through hash_expand_kernel, whose bound
    # (_code_bound_rank1_order) is what sees it here; the tables see it below
    rows, t0, t1 = _run_control(code_s, tsi, bound_one, T)

    # tables
    if mode == "deferred":
        assert "d_tables" not in one
        pend = one["pending"]
        assert pend["n_slots"] == T and pend["slots_are_timesteps"]
        assert torch.equal(pend["cw_slots"].double(), cw_t)
        g1 = pend["g_rank1"]
        # G per (slot, entry, f): K fl(w * dfeat) terms in float32 (merged runs or atomics): <= (K + 1) u A
        for s in range(T):
            b = U32 * (ref["K"][s][:, None].double() + 1) * ref["A"][s]
            _assert_within(g1[s], ref["G"][s], b, f"g_rank1 slot {s}")
            assert torch.equal((g1[s] != 0).any(1), ref["touched"][s]), f"touched entries of slot {s}"
            _assert_within(ch_g1[s], ref["G"][s], b, f"chunked g_rank1 slot {s}")
            _assert_within(g1[s], ch_g1[s], 2 * b, f"g_rank1 one vs chunks, slot {s}")
        del ch_g1
        one["d_tables"] = ops.rank1_expand(pend, E)
        del pend, g1
    del chunks
    _check_dense_tables(one["d_tables"], ref, cw_t, f"{mode}: d_tables")
    _check_dense_tables(ch_dense, ref, cw_t, f"{mode}: d_tables of the chunks")
    del ch_dense
    Gr, touched_r = _table_run_control(P.levels, saved, d_feat, rows, ref, cw_t, t0, t1)
    if mode == "deferred":     # the same run, seen in G: its contributions missing from slot t0
        b = U32 * (ref["K"][t0][:, None].double() + 1) * ref["A"][t0]
        _rejects(Gr, b, "a warp's run credited to the neighbouring timestep (G)")
    del Gr, touched_r

    # negative control on the tables: one sample's contribution at the finest hashed level removed
    idx, w = hashgrid_indices_weights(saved["xs"][s0:s0 + 1, :3].float(), P.levels)
    lines = idx[0, -1]                                                       # the 8 corners of level 15
    r, ab, k = dense_table_grad(ref["G"], ref["A"], ref["K"], cw_t, lines)
    contrib = w[0, -1].double()[:, None, None] * cw_t[tsi[s0]][None, :, None] * d_feat[s0, 30:].double()[None, None, :]
    _rejects(contrib, 2 * U32 * (k[:, None, None] + 2) * ab, "one sample's finest-level contribution removed")

    # the four modes against each other: two results each within its bound of the same float64 value are within the
    # sum of the bounds of each other (tables on a fixed sample of lines)
    g = torch.Generator(device=DEV).manual_seed(1)
    lines = torch.randperm(E, generator=g, device=DEV)[:1 << 16]
    r, ab, k = dense_table_grad(ref["G"], ref["A"], ref["K"], cw_t, lines)
    # (d_xs only between modes that blend the corner values the same way: the saved fp16 ones or the table's)
    mine = dict(codes=(one["d_blend_codes"].double(), bound_one),
                **{"d_xs_cv" if cv is not None else "d_xs_tab": (one["d_xs"].double(), dx_bound)},
                tables=(one["d_tables"][lines].double(), 2 * U32 * (k[:, None, None] + 2) * ab))
    for other, theirs in _MODES.items():
        for key, (val, bnd) in mine.items():
            if key in theirs:
                    _assert_within(val, theirs[key][0], bnd + theirs[key][1], f"{mode} vs {other}: {key}")
    _MODES[mode] = mine
    del ref


def test_per_sample_blend_codes_are_identical_across_chunks():
    """Component path (per-sample blend codes, direct scatter): d_sample_blend_codes and d_xs row for row."""
    P, NP, kw, tsi, saved, up = _batch()
    codes = NP.blend_codes[tsi].contiguous()

    from nersemble_b200 import ops
    one = ops.field_backward(NP, {k: saved[k] for k in ("sigma", "rgb", "feat", "xs")}, up["d_sigma"], up["d_rgb"],
                             window_hash=W_HASH, loss_scale=LS_FIELD, want_dx=True, want_tables=False,
                             sample_blend_codes=codes, **kw)
    parts = [ops.field_backward(NP, {k: saved[k][a:b] for k in ("sigma", "rgb", "feat", "xs")}, up["d_sigma"][a:b],
                                up["d_rgb"][a:b], window_hash=W_HASH, loss_scale=LS_FIELD, want_dx=True, want_tables=False,
                                sample_blend_codes=codes[a:b], **_rows_kw(kw, a, b)) for a, b in _chunks(N)]
    for name in ("d_sample_blend_codes", "d_xs", "d_feat"):
        assert torch.equal(torch.cat([p[name] for p in parts]), one[name]), name


# ---------------------------------------------------------------------------------------------------------------------
# more than 32 timesteps (d)
# ---------------------------------------------------------------------------------------------------------------------
PICKED = [0, 2, 3, 5, 8, 11, 12, 15, 19, 20, 24, 27, 29, 31, 34, 38, 40, 43, 45, 47]      # 20, not contiguous


def _picked_times(nt):
    g = torch.Generator().manual_seed(4)
    sel = torch.tensor(PICKED)[torch.randint(0, len(PICKED), (R_RAYS,), generator=g)]
    sel[:len(PICKED)] = torch.tensor(PICKED)
    return sel.float() / (nt - 1)


@pytest.mark.parametrize("which", ["20_of_48", "all_48"])
def test_more_than_32_timesteps(which):
    from nersemble_b200 import ops
    P, NP, kw, tsi, saved, up = _batch(T48, seed=23, time_of_ray=_picked_times if which == "20_of_48" else None, key=which)
    T, E = P.n_timesteps, P.levels.total_entries
    sc, bi = _scale_bias()
    uniq = torch.unique(tsi)
    if which == "20_of_48":
        assert uniq.tolist() == PICKED
        slot, n_slots = ops._rank1_slots(NP, DEV, kw)
        assert n_slots == 20 and torch.equal(slot[uniq].long(), torch.arange(20, device=DEV))   # not the identity
    else:
        assert uniq.numel() == 48 and ops._rank1_slots(NP, DEV, kw) == (None, 0)               # dense fallback
    mode = "rank1" if which == "20_of_48" else "direct"          # what field_backward(rank1=True) falls back to
    one = _field_bwd(NP, saved, up, kw, 0, N, "rank1")
    chunks = [_field_bwd(NP, saved, up, kw, a, b, "rank1") for a, b in _chunks(N)]
    assert torch.equal(torch.cat([c["d_feat"] for c in chunks]), one["d_feat"])
    assert torch.equal(torch.cat([c["d_xs"] for c in chunks]), one["d_xs"])
    d_feat = one["d_feat"]
    slot_map = torch.full((T,), -1, dtype=torch.long, device=DEV)
    slot_map[uniq] = torch.arange(uniq.numel(), device=DEV)
    ref = _hash_ref(P.levels, saved["xs"], d_feat, slot_map[tsi], uniq.numel())
    cw_t = cw16(NP.blend_codes, sc, bi)
    _check_dense_tables(one["d_tables"], ref, cw_t[uniq], f"{which}: d_tables")
    ch_dense = torch.stack([c.pop("d_tables") for c in chunks]).double().sum(0)
    _check_dense_tables(ch_dense, ref, cw_t[uniq], f"{which}: d_tables of the chunks")
    del ch_dense

    code_s, code_abs_s, _, _ = per_sample_terms(P.levels, saved["xs"], d_feat, NP.tables, cw_t[tsi], sc)
    code_t = torch.zeros((T, 32), dtype=torch.float64, device=DEV).index_add_(0, tsi, code_s)
    code_abs_t = torch.zeros_like(code_t).index_add_(0, tsi, code_abs_s)
    c_abs_t = torch.zeros_like(code_t).index_add_(0, tsi, code_s.abs())
    if mode == "rank1":
        bound_one = _code_bound_rank1_order(ref, NP.tables, sc, uniq, T)
        absent = [t for t in range(T) if t not in PICKED]
        assert (code_t[absent] == 0).all() and (one["d_blend_codes"][absent] == 0).all()
    else:
        bound_one = _code_bound_direct(code_abs_t, c_abs_t, tsi, N, T)
    bound_ch = _chunk_code_bounds(mode, P.levels, saved, d_feat, tsi, code_abs_s, code_s, NP.tables, sc, slot_map, uniq,
                                  uniq.numel(), T)
    ch_codes = torch.stack([c["d_blend_codes"] for c in chunks]).double()
    _check_codes(one["d_blend_codes"], ch_codes, code_t, bound_one, bound_ch, which)
    # one hash warp's run credited to the next timestep that occurs (in 20_of_48 also the next slot)
    rows, t0, t1 = _run_control(code_s, tsi, bound_one, T)
    _table_run_control(P.levels, saved, d_feat, rows, ref, cw_t[uniq], int(slot_map[t0]), int(slot_map[t1]))


# ---------------------------------------------------------------------------------------------------------------------
# deformation backward (e)
# ---------------------------------------------------------------------------------------------------------------------
def _deform_bwd(NP, saved, d_xs, kw, a, b, **extra):
    from nersemble_b200 import ops
    t0, t1 = a // 128, (b + 127) // 128
    s = {"deform_acts": saved["deform_acts"][t0:t1], "deform_enc": saved["deform_enc"][t0:t1]}
    return ops.deform_backward(NP, s, d_xs[a:b], window_deform=W_DEFORM, loss_scale=LS_DEFORM, **_rows_kw(kw, a, b), **extra)


@pytest.mark.parametrize("entry", ["table_codes", "sample_codes"])
def test_deform_backward_at_batch_scale(entry):
    """Both entry points of deform_bwd_kernel: warp codes indexed by timestep (d_warp_codes), and per-sample warp codes
    (component API, d_sample_warp_codes; here the timestep rows, per sample)."""
    P, NP, kw, tsi, saved, up = _batch()
    T = P.n_timesteps
    # a 16-row block that straddles two timesteps (deform_bwd_kernel's ts_uniform == false atomics) occurs
    blocks = tsi[: (N // 16) * 16].view(-1, 16)
    assert ((blocks != blocks[:, :1]).any(1)).sum() >= 10
    codes = NP.warp_codes[tsi].float().contiguous() if entry == "sample_codes" else None

    def run(a, b):
        extra = {} if codes is None else dict(sample_warp_codes=codes[a:b])
        g = _deform_bwd(NP, saved, up["d_xs"], kw, a, b, **extra)
        out = {**{f"d_stem_w{l}": g["d_stem_w"][l] for l in range(6)}, "d_stem_b": g["d_stem_b"], "d_r_w": g["d_r_w"],
               "d_v_w": g["d_v_w"], "d_r_b": g["d_r_b"], "d_v_b": g["d_v_b"]}
        # (per-sample rows copied out of their 65 536-row allocation, which one-tile launches would otherwise keep)
        out["codes"] = g["d_warp_codes"] if codes is None else g["d_sample_warp_codes"].clone()
        return out
    one = run(0, N)
    chunks = [run(a, b) for a, b in _chunks(N)]
    tiles = [run(a, min(N, a + 128)) for a in range(0, N, 128)]
    if codes is not None:      # (a) per-sample code gradients: row for row, in chunks and in one-tile launches
        assert torch.equal(torch.cat([c.pop("codes") for c in chunks]), one["codes"])
        assert torch.equal(torch.cat([t.pop("codes") for t in tiles]), one.pop("codes"))
    # d_warp_codes[t, col]: per 16-row block and layer (0, 4), one atomic when the block's rows share a timestep,
    # else one per row -- counted per timestep from the batch (chunks are whole tiles, so they count the same)
    blk = torch.arange(N, device=DEV) // 16
    mixed = torch.zeros(int(blk.max()) + 1, device=DEV).index_add_(0, blk, (tsi != tsi[blk * 16]).float()) > 0
    per_row = torch.where(mixed[blk], 2.0, 2.0 / 16).double()
    n_code_terms = torch.zeros(T, dtype=torch.float64, device=DEV).index_add_(0, tsi, per_row).ceil()[:, None]
    planted = [torch.zeros((), dtype=torch.float64, device=DEV)] * len(chunks)     # max planted / bound per chunk
    for name in one:
        t = torch.stack([x[name] for x in tiles]).double()
        exact, M = t.sum(0), t.abs().sum(0)
        ch = torch.stack([c[name] for c in chunks]).double()
        if name.startswith("d_stem"):
            # a tile's contribution is formed whole in one CTA (fragment scratch / shared-memory bias sums) and is
            # exact in a one-tile launch (x 1/loss_scale is exact); the one launch sums <= ceil(tiles / SMS) of them
            # per CTA (a store, then red.add) and then SMS CTAs (deform_dw_reduce_kernel / atomics), a chunk
            # CHUNK_TILES: |err| <= u (tiles_per_cta + SMS + CHUNK_TILES) M, M = sum over tiles of |contribution|,
            # + 8 for the float64 sum and second order
            bound = U32 * (math.ceil(N_TILES / SMS) + SMS + CHUNK_TILES + 8) * M
        elif name in ("d_r_w", "d_v_w"):
            # one atomic per tile and element, in any order (_any_order of the exact tile values)
            bound = U32 * (_any_order(t) + (CHUNK_TILES + 8) * M)
        elif name in ("d_r_b", "d_v_b"):
            # one atomic per warp, 8 per tile, in any order.  A one-tile value is the float32 sum of its 8 warp terms;
            # with each tile's terms taken as 8 equal parts the partial sums scale by at most 8 (_any_order of the tile
            # values x 8).  The tile values stand for the terms, which undercounts only where the 8 warp sums of a
            # tile cancel
            bound = U32 * (8 * _any_order(t) + (8 * CHUNK_TILES + 8) * M)
        else:
            # d_warp_codes: n_code_terms above, with the same caveat for the terms inside one tile
            bound = U32 * (n_code_terms + CHUNK_TILES + 8) * M
        _assert_within(one[name], exact, bound, f"{name}: one launch vs the sum of its tiles")
        _assert_within(ch.sum(0), exact, bound, f"{name}: chunked launches vs the sum of the tiles")
        _assert_within(one[name], ch.sum(0), 2 * bound, f"{name}: one launch vs chunked launches")
        # negative control per tensor: a chunk's tiles left out of the sum ("one tile per CTA dropped").  Every chunk
        # must be seen, except for the two 3-vectors d_r_b / d_v_b: their per-chunk sums of ~8 x 64 random-sign warp
        # terms can fall near zero in every component, which no float32 bound can tell from rounding; for them the
        # largest chunk must be seen, and every chunk is seen through the other tensors (below)
        r = torch.stack([(ch[k].abs() / (2 * bound).clamp_min(1e-300)).max() for k in range(ch.shape[0])])
        if name in ("d_r_b", "d_v_b"):
            _rejects(ch[int(r.argmax())], 2 * bound, f"{name} without its largest chunk")
        else:
            for k in range(ch.shape[0]):
                _rejects(ch[k], 2 * bound, f"{name} without chunk {k}")
        for k in range(ch.shape[0]):
            planted[k] = torch.maximum(planted[k], r[k])
    for k, r in enumerate(planted):
        assert r.item() >= 10.0, f"negative control: chunk {k} left out is only {r.item():.2f}x the bounds"
    if codes is None:
        assert one["codes"].abs().sum(1).ne(0).all()           # every timestep occurs in the batch


# ---------------------------------------------------------------------------------------------------------------------
# fused optimiser at the production table size (f)
# ---------------------------------------------------------------------------------------------------------------------
def test_table_adam_step_at_production_size():
    from nersemble_b200 import ops
    P, NP, kw, tsi, saved, up = _batch()
    grads = _field_bwd(NP, saved, up, kw, 0, N, "deferred")
    pend = grads["pending"]
    del grads
    E = P.levels.total_entries
    assert pend["n_slots"] == 24 and E > 6_000_000
    torch.cuda.empty_cache()
    p = P.tables.to(DEV).float().contiguous()
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    shadow = torch.empty(p.shape, dtype=torch.float16, device=DEV)
    ref = torch.nn.Parameter(p.clone())
    # eps 1e-8: the gradient is the float-atomic scatter's, and at eps = 1e-15 Adam turns the sign of a ~1e-12
    # residual into a full lr step (see test_fused_fields_adam_tracks_torch_adam_on_the_model)
    opt = torch.optim.Adam([ref], lr=5e-3, eps=1e-8, foreach=False)
    ref.grad = ops.rank1_expand(pend, E)
    opt.step()
    ref.grad = None
    ops.table_adam_step(p, m, v, shadow, step=1, lr=5e-3, eps=1e-8, pending=pend)
    del pend
    st = opt.state[ref]
    # tolerances of test_table_adam_step_matches_torch_adam (|got - want| <= atol + rtol |want|), in line blocks
    for a in range(0, E, 1 << 20):
        b = min(E, a + (1 << 20))
        for got, want, atol in ((m, st["exp_avg"], 1e-10), (v, st["exp_avg_sq"], 1e-20)):
            assert ((got[a:b] - want[a:b]).abs() <= atol + 2e-5 * want[a:b].abs()).all()
        assert (p[a:b] - ref.detach()[a:b]).abs().max().item() < 5e-3 * 1e-4
    assert torch.equal(shadow, p.half())
    moved = (p != P.tables.to(DEV)).flatten(1).any(1)
    assert moved.float().mean() > 0.3                             # a large share of the 6.3 M lines was updated
