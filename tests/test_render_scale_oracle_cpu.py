"""The host-side helpers of the render-scale GPU tests (tests/render_scale_oracle.py) on hand-worked cases: the tile ->
(CTA, iteration) map, the ragged-batch search, the chunker, the probe-tile selection, the float64 eval-mode composite
with its depth clip, and the reference-side mutations."""
import math

import pytest
import torch

import render_scale_oracle as rso
import scan_oracle as so


def test_tile_map_matches_the_persistent_schedule():
    # 10 tiles on 4 CTAs: CTA 0 runs tiles 0, 4, 8; CTA 1: 1, 5, 9; CTA 2: 2, 6; CTA 3: 3, 7
    n = 9 * 128 + 5
    assert rso.n_tiles(n) == 10 and rso.last_tile_rows(n) == 5 and rso.last_tile_rows(1280) == 128
    assert rso.tiles_per_cta(n, 4) == [3, 3, 2, 2]
    assert rso.tiles_per_cta(2 * 128, 4) == [1, 1, 0, 0]
    assert [rso.tile_place(t, 4) for t in (0, 5, 9, 7)] == [(0, 0), (1, 1), (1, 2), (3, 1)]
    assert all(rso.tile_of(*rso.tile_place(t, 132), 132) == t for t in range(1000))
    # every tile is run exactly once, by the CTA and iteration the map names
    for n, sms in ((n, 4), (8192 * 128, 132), (12345, 7)):
        mt = rso.tiles_per_cta(n, sms)
        runs = sorted(rso.tile_of(c, it, sms) for c in range(sms) for it in range(mt[c]))
        assert runs == list(range(rso.n_tiles(n)))


@pytest.mark.parametrize("sms", [132, 114, 7])
@pytest.mark.parametrize("last_rows,mod", [(1, 1), (65, -1)])
def test_ragged_batch_search(sms, last_rows, mod):
    R, S = rso.ragged_batch(sms, last_rows, mod, range(129, 256, 2))
    n = R * S
    assert S % 128 != 0
    assert rso.last_tile_rows(n) == last_rows and rso.n_tiles(n) % sms == mod % sms
    assert min(rso.tiles_per_cta(n, sms)) >= 8
    # the smallest such batch over the candidate counts
    for S2 in range(129, 256, 2):
        for R2 in range(1, R * S // S2 + 1):
            n2 = R2 * S2
            if n2 < n and min(rso.tiles_per_cta(n2, sms)) >= 8:
                assert not (rso.last_tile_rows(n2) == last_rows and rso.n_tiles(n2) % sms == mod % sms), (R2, S2)


def test_chunker():
    counts = torch.tensor([3, 5, 0, 2, 8, 1, 1, 0])
    ch = rso.chunk_rays(counts, 8)
    assert ch == [(0, 3), (3, 4), (4, 5), (5, 8)]
    assert ch[0][0] == 0 and ch[-1][1] == 8 and all(a[1] == b[0] for a, b in zip(ch, ch[1:]))
    assert all(int(counts[a:b].sum()) <= 8 for a, b in ch)
    assert rso.chunk_rays(torch.full((10,), 256), 64 * 128) == [(0, 10)]
    assert rso.chunk_rays(torch.full((100,), 256), 8192) == [(0, 32), (32, 64), (64, 96), (96, 100)]
    with pytest.raises(ValueError):
        rso.chunk_rays(torch.tensor([1, 9]), 8)


def test_probe_tiles_and_ray_selection():
    sms, S = 4, 96
    n = 50 * S                             # 4800 samples: 38 tiles, the last one 64 rows; CTAs run 10, 10, 9, 9
    tiles = rso.probe_tiles(n, sms, n_spread=2)
    labels = dict((t, lab) for lab, t in tiles)
    assert tiles[0] == ("ragged last tile", 37)
    for c, its in ((0, (2, 3, 8, 9)), (1, (2, 3)), (3, (2, 3, 7, 8))):
        for it in its:
            assert rso.tile_of(c, it, sms) in labels, (c, it)
    assert len(labels) == len(tiles)       # no tile twice
    ri = torch.arange(50).repeat_interleave(S)
    rays, taken = rso.select_rays(ri, tiles, max_rays=6, extra=[0])
    # tile 37 = samples 4736..4799 = ray 49; each further tile adds at most 2 rays
    assert 0 in rays.tolist() and 49 in rays.tolist() and rays.numel() <= 6
    for _, t in taken:
        assert set(torch.unique(ri[t * 128:(t + 1) * 128]).tolist()) <= set(rays.tolist())
    info = torch.stack([torch.arange(50) * S, torch.full((50,), S)], -1)
    idx, sub, local = rso.subset_samples(info, torch.tensor([2, 5]))
    assert torch.equal(idx, torch.cat([torch.arange(2 * S, 3 * S), torch.arange(5 * S, 6 * S)]))
    assert torch.equal(sub, torch.tensor([[0, S], [S, S]])) and torch.equal(local, torch.arange(2).repeat_interleave(S))


def test_ordered_float_map():
    import struct
    vals = [float(torch.tensor(f, dtype=torch.float32)) for f in (-3.4e38, -2.25, -1e-40, -0.0, 0.0, 1e-40, 1.5, 7.0, 3.4e38)]
    encs = []
    for f in vals:
        u = struct.unpack("<I", struct.pack("<f", f))[0]
        enc = (~u & 0xffffffff) if (u & 0x80000000) else (u | 0x80000000)   # float_to_ordered
        assert rso.ordered_to_float(enc) == f
        encs.append(enc)
    assert encs == sorted(encs)                                              # unsigned order is float order


def test_eval_composite_by_hand():
    """Two rays of two samples, dt = 0.5: ray 0 sigma (2, 4), ray 1 sigma (0, 0); and one empty ray."""
    info = torch.tensor([[0, 2], [2, 2], [4, 0]])
    ts = torch.tensor([1.0, 1.5, 3.0, 3.5]); te = ts + 0.5
    sigma = torch.tensor([2.0, 4.0, 0.0, 0.0])
    rgb = torch.tensor([[0.5, float("nan"), 3.0], [0.25, 0.5, -1.0], [0.1, 0.2, 0.3], [0.9, 0.8, 0.7]])
    off = torch.tensor([[1.0, 0, 0], [0, 2.0, 0], [5.0, 5.0, 5.0], [1.0, 1.0, 1.0]])
    out = rso.composite_eval(info, ts, te, sigma, rgb, off)
    e1, e2 = math.exp(-1.0), math.exp(-2.0)
    w = [1 - e1, e1 * (1 - e2), 0.0, 0.0]
    assert torch.allclose(out["weights"], torch.tensor(w, dtype=torch.float64), rtol=1e-15, atol=0)
    acc0 = w[0] + w[1]
    assert torch.allclose(out["accumulation"], torch.tensor([acc0, 0.0, 0.0], dtype=torch.float64), rtol=1e-15, atol=0)
    raw = [w[0] * 0.5 + w[1] * 0.25 + 1 - acc0, w[0] * 0.0 + w[1] * 0.5 + 1 - acc0, w[0] * 3.0 - w[1] + 1 - acc0]
    want_rgb = torch.tensor([[min(max(v, 0.0), 1.0) for v in raw], [1.0] * 3, [1.0] * 3], dtype=torch.float64)
    assert torch.allclose(out["rgb"], want_rgb, rtol=1e-15, atol=1e-15)
    assert out["rgb"][0, 2] == 1.0 and raw[2] > 1.0                       # clamped
    # expected depth: midpoints 1.25, 1.75; ray 1 has no weight -> 0, clipped up to the lowest midpoint 1.25
    d0 = (w[0] * 1.25 + w[1] * 1.75) / (acc0 + 1e-10)
    assert out["clip"] == (1.25, 3.75)
    assert torch.allclose(out["depth"], torch.tensor([d0, 1.25, 1.25], dtype=torch.float64), rtol=1e-15, atol=0)
    clipped = rso.composite_eval(info, ts, te, sigma, rgb, off, clip=(1.6, 2.0))
    assert torch.allclose(clipped["depth"], torch.tensor([max(d0, 1.6), 1.6, 1.6], dtype=torch.float64))
    want_def = torch.tensor([[w[0], 2 * w[1], 0.0], [0.0] * 3, [0.0] * 3], dtype=torch.float64)
    assert torch.allclose(out["deformation"], want_def, rtol=1e-15, atol=0)
    assert torch.equal(out["deformation_scale"][1:], torch.zeros(2, 3, dtype=torch.float64))   # zero weights: exact 0
    assert (out["deformation_scale"][0, :2] > 0).all() and out["deformation_scale"][0, 2] == 0
    assert rso.midpoint_range(ts, te) == (1.25, 3.75) and rso.midpoint_range(ts[:0], te[:0]) is None
    # the float32 bound of error_constant holds for a float32 evaluation of the same composite
    ref = so.composite(info, ts, te, sigma, torch.nan_to_num(rgb))
    assert torch.equal(ref["weights"], out["weights"])


def test_mutations_and_ratios():
    sms, n = 3, 10 * 128 + 7
    v = torch.arange(n, dtype=torch.float32)
    s = rso.stale_tile(v, 10, sms, n)                    # the ragged tile 10 (7 rows) gets tile 4's first 7 rows
    assert torch.equal(s[1280:], torch.arange(512, 519, dtype=torch.float32)) and torch.equal(s[:1280], v[:1280])
    with pytest.raises(AssertionError):
        rso.stale_tile(v, 5, sms, n)
    h = rso.shift_tile_rows(v, 2, n)
    assert torch.equal(h[256:383], v[257:384]) and h[383] == v[383] and torch.equal(h[:256], v[:256])
    assert rso.bound_ratio(torch.tensor([1.0, 2.0]), torch.tensor([1.0, 2.5]), torch.tensor([1.0, 0.1])) == pytest.approx(5.0)
    assert rso.bound_ratio(torch.tensor([1.0]), torch.tensor([2.0]), torch.tensor([0.0])) == math.inf
    assert rso.bound_ratio(torch.tensor([1.0]), torch.tensor([1.0]), torch.tensor([0.0])) == 0.0
    assert rso.tol_ratio(torch.tensor([1.1]), torch.tensor([1.0]), 0.0, 0.05) == pytest.approx(2.0)
