"""The float64 references of backward_scale_oracle against torch autograd through oracle.pipeline.hash_ensemble
(Precision "none": fp16-stored tables, all math in float64 here), on CPU: the dense table gradient (from G), the
time-code gradient (from G and per sample) and the position gradient."""
import pytest
import torch

from backward_scale_oracle import (code_grad_from_G, cw16, dense_table_grad, hash_scatter_ref, per_sample_terms)
from oracle import pipeline as pl
from oracle.tp.tcnn_cpu import Precision


@pytest.fixture(autouse=True)
def _mode():
    Precision.mode = "none"; Precision.autocast = False
    yield
    Precision.mode = "reference"


def _batch(T=4, n=300, seed=3):
    P = pl.random_params(seed=seed, n_timesteps=T, log2_hashmap_size=12, table_scale=0.5, time_std_scale=100.0)
    g = torch.Generator().manual_seed(seed)
    x = torch.rand((n, 3), generator=g)
    x[:7] = torch.rand((7, 3), generator=g) * 1e-3          # near the lower faces
    sel = torch.ones(n); sel[::23] = 0                       # outside the box: coordinates zeroed, selector 0
    x = x * sel[:, None]
    xs = torch.cat([x, sel[:, None]], -1)
    ts = torch.randint(0, T, (n,), generator=g)              # ragged: unsorted, uneven per timestep
    ts[:50] = 1
    d_feat = torch.randn((n, 32), generator=g)
    sc = (torch.rand(32, generator=g) * 0.5 + 0.5).tolist()  # a window-like per-member scale, zero bias
    return P, xs, ts, d_feat, sc


def _rel(got, want):
    return ((got - want).abs().max() / want.abs().max()).item()


def test_references_match_float64_autograd_through_the_oracle():
    T = 4
    P, xs, ts, d_feat, sc = _batch(T)
    lv, n = P.levels, xs.shape[0]
    cw_t = cw16(P.time_emb, sc, [0.0] * 32)                          # [T, 32], fp16 values
    tables64 = P.tables.half().double().requires_grad_(True)         # the fp16 table, differentiated in float64
    codes = cw_t[ts].clone().requires_grad_(True)                    # per-sample blend weights (already fp16 values)
    x = xs[:, :3].clone().requires_grad_(True)
    P.tables = tables64
    out = pl.hash_ensemble(P, x, codes, None)                        # [n, 32] (row d = level * 2 + f)
    (out * d_feat.double()).sum().backward()

    G, A, K, touched = hash_scatter_ref(lv, xs, d_feat, ts, T)
    lines = torch.arange(lv.total_entries)
    dense, dense_abs, _ = dense_table_grad(G, A, K, cw_t, lines)
    assert _rel(dense, tables64.grad) < 1e-12
    assert torch.equal(touched.any(0), (tables64.grad != 0).any(-1).any(-1))
    assert (dense.abs() <= dense_abs * (1 + 1e-12)).all()

    V = P.tables.detach().half()
    code, code_abs, dxs, dxs_abs = per_sample_terms(lv, xs, d_feat, V, cw_t[ts], sc)
    sc64 = torch.tensor(sc, dtype=torch.float32).double()
    assert _rel(code, codes.grad * sc64) < 1e-12                     # dL/dcode = dL/dcw * cw_scale
    per_t = torch.zeros((T, 32), dtype=torch.float64).index_add_(0, ts, code)
    assert _rel(code_grad_from_G(G, V, sc), per_t) < 1e-12           # the rank-1 route gives the same sums
    assert (code.abs() <= code_abs * (1 + 1e-12)).all()
    # the oracle's trilinear weights are float32 tensors, so autograd rounds dL/dw to float32 before the chain to x:
    # agreement to float32 precision, not float64
    want_dx = x.grad.double() * xs[:, 3:4].double()
    assert _rel(dxs, want_dx) < 1e-6
    assert (dxs[xs[:, 3] == 0] == 0).all()
    assert (dxs.abs() <= dxs_abs * (1 + 1e-12)).all()


def test_slots_and_saved_corner_values():
    """A slot map that is not the identity puts each timestep's sum in its slot; the saved-corner form of d_xs equals
    the table form when the corner values are the blended table values."""
    T = 6
    P, xs, ts, d_feat, sc = _batch(T, n=200, seed=5)
    ts = ts.clamp(max=T - 1); ts[ts == 2] = 4                    # timesteps 0, 1, 3, 4, 5 occur; 2 does not
    lv = P.levels
    slot = torch.full((T,), -1, dtype=torch.long)
    uniq = torch.unique(ts)
    slot[uniq] = torch.arange(uniq.numel())
    G, A, K, touched = hash_scatter_ref(lv, xs, d_feat, slot[ts], uniq.numel())
    Gi, Ai, Ki, _ = hash_scatter_ref(lv, xs, d_feat, ts, T)
    assert torch.equal(G, Gi[uniq]) and torch.equal(A, Ai[uniq]) and torch.equal(K, Ki[uniq])
    assert (Ki[2] == 0).all()

    from oracle.tp.tcnn_cpu import hashgrid_indices_weights
    V = P.tables.half()
    cw_t = cw16(P.time_emb, sc, [0.0] * 32)
    idx, _ = hashgrid_indices_weights(xs[:, :3], lv)
    blended = torch.einsum("nlcmf,nm->nlcf", V[idx].double(), cw_t[ts])
    _, _, dx_tab, _ = per_sample_terms(lv, xs, d_feat, V, cw_t[ts], sc)
    _, _, dx_cv, _ = per_sample_terms(lv, xs, d_feat, V, cw_t[ts], sc, corner_vals=blended)
    assert _rel(dx_cv, dx_tab) < 1e-12
