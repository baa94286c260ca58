"""Gradients of the stand-alone component modules (HashEnsemble, SE3DeformationField, NeRSembleNeRFactoField) vs
autograd through the CPU oracle ("kernel" precision mode), and vs the table-indexed training backward."""
import pytest
import torch

from conftest import native_from_oracle, oracle_params
from oracle import pipeline as pl
from oracle.tp.tcnn_cpu import Precision, half_round, hashgrid_indices_weights

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TRAINED = dict(seed=19980801, n_timesteps=4, log2_hashmap_size=14, table_scale=0.5, time_std_scale=100.0,
               deform_last_scale=1e-3)
DEFORM = dict(TRAINED, deform_last_scale=0.05)          # |r| above the 1e-2 clamp: exercises d theta / d r
N = 700                                                  # ragged: 5 full tiles + 60


@pytest.fixture(autouse=True)
def _mode():
    Precision.mode = "kernel"; Precision.autocast = False
    yield
    Precision.mode = "reference"


def _relerr(got, want):
    return ((got.detach().cpu() - want).abs().max() / want.abs().max().clamp_min(1e-30)).item()


def _check_tables(got, want):
    got = got.detach().cpu()
    assert _relerr(got, want) < 8e-2
    assert ((got != 0) == (want != 0)).float().mean() > 0.999
    cos = torch.nn.functional.cosine_similarity(got.reshape(1, -1), want.reshape(1, -1)).item()
    assert cos > 0.9995, cos


def _hash_ensemble(P, disable_initial):
    from nersemble_b200.plugin.components import HashEnsemble, HashEnsembleConfig, TCNNHashEncodingConfig
    he = HashEnsemble(HashEnsembleConfig(32, TCNNHashEncodingConfig(log2_hashmap_size=14), disable_initial, True)).to(DEV)
    assert he.tables.shape == P.tables.shape
    with torch.no_grad():
        he.tables.copy_(P.tables)
    return he


def _deformation_field(P):
    from nersemble_b200.plugin.components import SE3DeformationField, SE3DeformationFieldConfig
    de = SE3DeformationField(P.aabb.clone(), SE3DeformationFieldConfig(warp_code_dim=128)).to(DEV)
    f = de.se3_field
    with torch.no_grad():
        for l, layer in enumerate(f.mlp_stem.layers):
            layer.weight.copy_(P.deform_w[l]); layer.bias.copy_(P.deform_b[l])
        f.mlp_r.layers[0].weight.copy_(P.r_w); f.mlp_r.layers[0].bias.copy_(P.r_b)
        f.mlp_v.layers[0].weight.copy_(P.v_w); f.mlp_v.layers[0].bias.copy_(P.v_b)
    return de


def _field(P):
    from nersemble_b200.plugin.components import HashEnsembleConfig, TCNNHashEncodingConfig
    from nersemble_b200.plugin.field import NeRSembleNeRFactoField
    f = NeRSembleNeRFactoField(P.aabb.clone(), 16, use_hash_ensemble=True, spherical_harmonics_degree=0,
                               hash_ensemble_config=HashEnsembleConfig(32, TCNNHashEncodingConfig(log2_hashmap_size=14),
                                                                       True, True)).to(DEV)
    with torch.no_grad():
        f.hash_ensemble.tables.copy_(P.tables)
        f.mlp_base.params.copy_(torch.cat([w.reshape(-1) for w in P.base_w]))
        f.mlp_head.params.copy_(torch.cat([w.reshape(-1) for w in P.head_w]))
    return f


def _ray_samples(positions, directions, time_codes):
    from nersemble_b200.nerfstudio_shim import Frustums, RaySamples
    n = positions.shape[0]
    z = torch.zeros((n, 1), device=positions.device)
    return RaySamples(Frustums(positions, directions, z, z, None), camera_indices=torch.zeros((n, 1), dtype=torch.long,
                      device=positions.device), metadata={"time_codes": time_codes})


def _blend_oracle(P, x, codes, window, disable_initial):
    """HashEnsemble.forward in kernel precision with the blend options of the module (pl.hash_ensemble fixes them)."""
    idx, w = hashgrid_indices_weights(x, P.levels)
    tab = half_round(P.tables)
    code, win = pl.blend_code(P, codes, window, disable_initial, True)
    cw = code if win is None else code * win[None, :]
    S, L = x.shape[0], P.levels.n_levels
    out = torch.zeros(S, L, 2)
    for c in range(8):
        vals = tab[idx[:, :, c].reshape(-1)].view(S, L, 32, 2)
        out = out + w[:, :, c, None] * (vals * cw[:, None, :, None]).sum(2)
    return out.reshape(S, L * 2)


@pytest.mark.parametrize("disable_initial", [True, False])
@pytest.mark.parametrize("window", [1.0, 1.5, 20.25, 32.0])
def test_hash_ensemble_grads_vs_oracle(window, disable_initial):
    P = oracle_params(TRAINED)
    g = torch.Generator().manual_seed(11)
    x = torch.rand((N, 3), generator=g)
    codes = torch.randn((N, 32), generator=g) * 0.2
    g_out = torch.randn((N, 32), generator=g)
    P.tables.requires_grad_(True); P.tables.grad = None
    xo, co = x.clone().requires_grad_(True), codes.clone().requires_grad_(True)
    (_blend_oracle(P, xo, co, window, disable_initial) * g_out).sum().backward()
    P.tables.requires_grad_(False)

    he = _hash_ensemble(P, disable_initial)
    xg, cg = x.to(DEV).requires_grad_(True), codes.to(DEV).requires_grad_(True)
    out = he(xg, cg, window_hash_encodings=window)
    with torch.no_grad():
        assert torch.equal(out, he(xg, cg, window_hash_encodings=window))      # grad-enabled forward is the same call
    (out.float() * g_out.to(DEV)).sum().backward()
    _check_tables(he.tables.grad, P.tables.grad)
    if window == 1.0 and disable_initial:       # the reference replaces the code with ones: no code gradient at all
        assert co.grad is None and (cg.grad == 0).all()
    else:
        assert _relerr(cg.grad, co.grad) < 2e-2
    assert _relerr(xg.grad, xo.grad) < 3e-2


def _deform_case(n=N, seed=9):
    P = oracle_params(DEFORM)
    g = torch.Generator().manual_seed(seed)
    lo, hi = P.aabb[0], P.aabb[1]
    pos = lo + (torch.rand((n, 3), generator=g) * 0.9 + 0.05) * (hi - lo)
    tsteps = torch.sort(torch.randint(0, 4, (n,), generator=g))[0]
    return P, g, pos, tsteps


def _deform_param_grads(de):
    f = de.se3_field
    return ([l.weight.grad for l in f.mlp_stem.layers], [l.bias.grad for l in f.mlp_stem.layers],
            f.mlp_r.layers[0].weight.grad, f.mlp_r.layers[0].bias.grad, f.mlp_v.layers[0].weight.grad,
            f.mlp_v.layers[0].bias.grad)


@pytest.mark.parametrize("w_deform", [5.5, None])
def test_deformation_field_grads_vs_oracle(w_deform):
    P, g, pos, _ = _deform_case()
    codes = torch.randn((N, 128), generator=g) * 0.1       # a distinct warp code per sample
    g_off = torch.randn((N, 3), generator=g)
    for t in P.all_tensors():
        t.grad = None
    P.requires_grad_(True)
    co = codes.clone().requires_grad_(True)
    (pl.compute_offsets(P, pos, co, w_deform) * g_off).sum().backward()
    P.requires_grad_(False)

    de = _deformation_field(P)
    cg = codes.to(DEV).requires_grad_(True)
    off = de.compute_offsets(pos.to(DEV), cg, w_deform)
    with torch.no_grad():
        assert torch.equal(off, de.compute_offsets(pos.to(DEV), cg, w_deform))
    (off * g_off.to(DEV)).sum().backward()
    sw, sb, rw, rb, vw, vb = _deform_param_grads(de)
    for l in range(6):
        assert _relerr(sw[l], P.deform_w[l].grad) < 4e-2, l
        assert _relerr(sb[l], P.deform_b[l].grad) < 4e-2, l
    assert _relerr(rw, P.r_w.grad) < 3e-2 and _relerr(vw, P.v_w.grad) < 3e-2
    assert _relerr(rb, P.r_b.grad) < 3e-2 and _relerr(vb, P.v_b.grad) < 3e-2
    assert _relerr(cg.grad, co.grad) < 4e-2


def test_deformation_per_sample_codes_match_the_table_path():
    """Codes gathered from a [T,128] table: the per-sample code gradients summed by timestep and every parameter
    gradient equal the table-indexed training backward's."""
    from nersemble_b200 import ops
    P, g, pos, tsteps = _deform_case()
    times = tsteps.float() / 3
    g_off = torch.randn((N, 3), generator=g).to(DEV)
    w_deform = 5.5
    de = _deformation_field(P)
    codes = P.time_emb_deform[tsteps].to(DEV).requires_grad_(True)
    (de.compute_offsets(pos.to(DEV), codes, w_deform) * g_off).sum().backward()

    NP = native_from_oracle(P, DEV)
    kw = dict(positions=pos.to(DEV), sample_times=times.to(DEV))
    saved = ops.field_forward(NP, window_hash=None, window_deform=w_deform, use_deformation=True,
                              want=("offsets", "deform_acts"), **kw)
    aabb = P.aabb.to(DEV)
    ref = ops.deform_backward(NP, saved, g_off * (aabb[1] - aabb[0]), window_deform=w_deform,
                              loss_scale=de.mlp_loss_scale, **kw)
    summed = torch.zeros((4, 128), device=DEV).index_add_(0, tsteps.to(DEV), codes.grad)
    assert _relerr(summed, ref["d_warp_codes"].cpu()) < 1e-4
    sw, sb, rw, rb, vw, vb = _deform_param_grads(de)
    for l in range(6):
        assert _relerr(sw[l], ref["d_stem_w"][l].cpu()) < 1e-4, l
        assert _relerr(sb[l], ref["d_stem_b"][l].cpu()) < 1e-4, l
    for got, key in ((rw, "d_r_w"), (rb, "d_r_b"), (vw, "d_v_w"), (vb, "d_v_b")):
        assert _relerr(got, ref[key].cpu()) < 1e-4, key


def _field_case():
    P = oracle_params(TRAINED)
    g = torch.Generator().manual_seed(5)
    lo, hi = P.aabb[0], P.aabb[1]
    pos = lo + (torch.rand((N, 3), generator=g) * 1.1 - 0.05) * (hi - lo)     # a few outside the box
    dirs = torch.randn((N, 3), generator=g); dirs = dirs / dirs.norm(dim=-1, keepdim=True)
    tsteps = torch.sort(torch.randint(0, 4, (N,), generator=g))[0]
    return P, g, pos, dirs, tsteps


@pytest.mark.parametrize("entry", ["forward", "density_fn"])
def test_field_grads_vs_oracle(entry):
    from nersemble_b200.nerfstudio_shim import FieldHeadNames
    P, g, pos, dirs, tsteps = _field_case()
    codes = P.time_emb[tsteps]
    w_hash = 20.25
    g_sigma = torch.randn((N,), generator=g) * 0.1
    g_rgb = torch.randn((N, 3), generator=g)
    for t in P.all_tensors():
        t.grad = None
    P.requires_grad_(True)
    po, co = pos.clone().requires_grad_(True), codes.detach().clone().requires_grad_(True)
    sigma, geo = pl.field_density(P, po, co, w_hash)
    loss = (sigma[:, 0] * g_sigma).sum()
    if entry == "forward":
        loss = loss + (pl.field_rgb(P, dirs, geo) * g_rgb).sum()
    loss.backward()
    P.requires_grad_(False)

    f = _field(P)
    pg, cg = pos.to(DEV).requires_grad_(True), codes.detach().to(DEV).requires_grad_(True)
    if entry == "forward":
        run = lambda: f(_ray_samples(pg, dirs.to(DEV), cg), window_hash_encodings=w_hash)
        out = run()
        with torch.no_grad():
            ref = run()
        for k in (FieldHeadNames.RGB, FieldHeadNames.DENSITY):
            assert torch.equal(out[k], ref[k])
        loss = (out[FieldHeadNames.DENSITY][:, 0] * g_sigma.to(DEV)).sum() + (out[FieldHeadNames.RGB] * g_rgb.to(DEV)).sum()
    else:
        sig = f.density_fn(pg, None, w_hash, cg)
        with torch.no_grad():
            assert torch.equal(sig, f.density_fn(pg, None, w_hash, cg))
        loss = (sig[:, 0] * g_sigma.to(DEV)).sum()
    loss.backward()
    # density alone: the smaller gradient carries relatively more of the fp16-delta error than with the colour term
    assert _relerr(pg.grad, po.grad) < (3e-2 if entry == "forward" else 5e-2)
    pn = (pos - P.aabb[0]) / (P.aabb[1] - P.aabb[0])
    outside = ~((pn > 0) & (pn < 1)).all(-1)
    assert outside.any() and (pg.grad.cpu()[outside] == 0).all()
    assert _relerr(f.mlp_base.params.grad, torch.cat([w.grad.reshape(-1) for w in P.base_w])) < 2e-2
    if entry == "forward":
        assert _relerr(f.mlp_head.params.grad, torch.cat([w.grad.reshape(-1) for w in P.head_w])) < 2e-2
    # one sample's code gradient sums few fp16-delta contributions, like one table entry's (the training test's 2e-2
    # bound is for per-timestep sums): the per-entry bound
    assert _relerr(cg.grad, co.grad) < 8e-2
    _check_tables(f.hash_ensemble.tables.grad, P.tables.grad)

    # per-sample code gradients summed by timestep == the table-indexed backward's d_blend_codes
    from nersemble_b200 import ops
    NP = native_from_oracle(P, DEV)
    kw = dict(positions=pos.to(DEV), sample_times=(tsteps.float() / 3).to(DEV), sample_directions=dirs.to(DEV))
    saved = ops.field_forward(NP, window_hash=w_hash, use_deformation=False, want=("sigma", "rgb", "feat", "xs"), **kw)
    ref = ops.field_backward(NP, saved, g_sigma.to(DEV), g_rgb.to(DEV) if entry == "forward" else None,
                             window_hash=w_hash, loss_scale=f.mlp_loss_scale, rank1=False, **kw)
    summed = torch.zeros((4, 32), device=DEV).index_add_(0, tsteps.to(DEV), cg.grad)
    assert _relerr(summed, ref["d_blend_codes"].cpu()) < 1e-3


def _composite(sigma, rgb, ts, te, ri, n_rays):
    """Alpha compositing of packed samples on a white background, in plain torch (both devices)."""
    sd = sigma * (te - ts)
    inc = torch.cumsum(sd, 0)
    cnt = torch.zeros(n_rays, dtype=torch.long, device=sd.device).index_add_(0, ri, torch.ones_like(ri))
    first = torch.cumsum(cnt, 0) - cnt
    before = torch.cat([torch.zeros(1, device=sd.device), inc])[first][ri]
    trans = torch.exp(-(inc - sd - before))
    w = trans * (1 - torch.exp(-sd))
    comp = torch.zeros((n_rays, 3), device=sd.device).index_add_(0, ri, w[:, None] * rgb)
    acc = torch.zeros((n_rays,), device=sd.device).index_add_(0, ri, w)
    return comp + (1 - acc)[:, None]


def test_deformation_field_then_field_then_compositing_vs_oracle():
    """deformation_field.forward -> field.forward -> torch compositing on packed samples: every model parameter and
    both time embeddings get the oracle's gradients."""
    from nersemble_b200.nerfstudio_shim import FieldHeadNames
    P = oracle_params(DEFORM)
    for t in P.all_tensors():
        t.grad = None
    g = torch.Generator().manual_seed(21)
    R, n_per = 24, 40
    o = torch.tensor([[0.0, 0.0, 4.0]]).repeat(R, 1) + torch.randn((R, 3), generator=g) * 0.2
    tgt = torch.rand((R, 3), generator=g) * 2 - 1
    d = tgt - o; d = d / d.norm(dim=-1, keepdim=True)
    ts, te, ri = pl.fixed_samples(o, d, P.aabb, n_per, 0.05, near=0.2)
    tsteps = torch.randint(0, 4, (R,), generator=g)[ri]
    w_hash, w_deform = 20.25, 5.5
    g_comp = torch.randn((R, 3), generator=g)

    P.requires_grad_(True)
    pos = o[ri] + d[ri] * ((ts + te)[:, None] / 2)
    off = pl.compute_offsets(P, pos, P.time_emb_deform[tsteps], w_deform)
    sigma, geo = pl.field_density(P, pos + off, P.time_emb[tsteps], w_hash)
    rgb = pl.field_rgb(P, d[ri], geo)
    (_composite(sigma[:, 0], rgb, ts, te, ri, R) * g_comp).sum().backward()
    P.requires_grad_(False)

    from nersemble_b200.nerfstudio_shim import Frustums, RaySamples
    de, f = _deformation_field(P), _field(P)
    emb = torch.nn.Parameter(P.time_emb.to(DEV)); emb_d = torch.nn.Parameter(P.time_emb_deform.to(DEV))
    tg, rg = tsteps.to(DEV), ri.to(DEV)
    n = ts.shape[0]
    rs = RaySamples(Frustums(o.to(DEV)[rg], d.to(DEV)[rg], ts.to(DEV)[:, None], te.to(DEV)[:, None], None),
                    camera_indices=torch.zeros((n, 1), dtype=torch.long, device=DEV), metadata={"time_codes": emb[tg]})
    rs = de(rs, emb_d[tg], w_deform)
    rs.frustums.offsets.retain_grad()
    out = f(rs, window_hash_encodings=w_hash)
    comp = _composite(out[FieldHeadNames.DENSITY][:, 0], out[FieldHeadNames.RGB], ts.to(DEV), te.to(DEV), rg, R)
    (comp * g_comp.to(DEV)).sum().backward()

    assert _relerr(emb.grad, P.time_emb.grad) < 3e-2
    assert _relerr(emb_d.grad, P.time_emb_deform.grad) < 6e-2
    assert _relerr(f.mlp_base.params.grad, torch.cat([w.grad.reshape(-1) for w in P.base_w])) < 3e-2
    assert _relerr(f.mlp_head.params.grad, torch.cat([w.grad.reshape(-1) for w in P.head_w])) < 3e-2
    _check_tables(f.hash_ensemble.tables.grad, P.tables.grad)
    # Deformation parameters: the oracle's deformation backward seeded with the offset gradient the field produced.
    # (End to end, the few-percent per-sample error of the field's position gradient survives into sums over samples
    # that largely cancel -- 13 % on the last stem layer -- and would hide what this checks: the hand-over between
    # the two modules.)
    g_off = rs.frustums.offsets.grad.cpu()
    for t in P.all_tensors():
        t.grad = None
    P.requires_grad_(True)
    (pl.compute_offsets(P, pos, P.time_emb_deform[tsteps], w_deform) * g_off).sum().backward()
    P.requires_grad_(False)
    sw, sb, rw, rb, vw, vb = _deform_param_grads(de)
    for l in range(6):
        assert _relerr(sw[l], P.deform_w[l].grad) < 4e-2, l
        assert _relerr(sb[l], P.deform_b[l].grad) < 4e-2, l
    for got, want in ((rw, P.r_w), (rb, P.r_b), (vw, P.v_w), (vb, P.v_b)):
        assert _relerr(got, want.grad) < 3e-2
    assert _relerr(emb_d.grad, P.time_emb_deform.grad) < 4e-2


def test_empty_batches_give_empty_or_zero_gradients():
    P = oracle_params(DEFORM)
    he, de, f = _hash_ensemble(P, True), _deformation_field(P), _field(P)
    x = torch.zeros((0, 3), device=DEV, requires_grad=True)
    c = torch.zeros((0, 32), device=DEV, requires_grad=True)
    he(x, c, window_hash_encodings=20.25).float().sum().backward()
    assert x.grad.shape == (0, 3) and c.grad.shape == (0, 32) and not he.tables.grad.any()
    wc = torch.zeros((0, 128), device=DEV, requires_grad=True)
    de.compute_offsets(torch.zeros((0, 3), device=DEV), wc, 5.5).sum().backward()
    assert wc.grad.shape == (0, 128) and not de.se3_field.mlp_stem.layers[0].weight.grad.any()
    p = torch.zeros((0, 3), device=DEV, requires_grad=True)
    f.density_fn(p, None, 20.25, torch.zeros((0, 32), device=DEV)).sum().backward()
    assert p.grad.shape == (0, 3) and not f.mlp_base.params.grad.any() and not f.hash_ensemble.tables.grad.any()


def test_fused_adam_steps_a_component_table_gradient_like_torch_adam():
    from nersemble_b200.optim import FusedFieldsAdam
    P = oracle_params(TRAINED)
    g = torch.Generator().manual_seed(4)
    x, c = torch.rand((N, 3), generator=g).to(DEV), (torch.randn((N, 32), generator=g) * 0.2).to(DEV)
    g_out = torch.randn((N, 32), generator=g).to(DEV)
    he = _hash_ensemble(P, True)
    (he(x, c, window_hash_encodings=20.25).float() * g_out).sum().backward()
    assert he.tables.grad is not None and he.tables.grad.any()
    ref = torch.nn.Parameter(he.tables.detach().clone())
    ref.grad = he.tables.grad.clone()
    FusedFieldsAdam([he.tables], lr=5e-3, eps=1e-15).step()
    torch.optim.Adam([ref], lr=5e-3, eps=1e-15).step()
    torch.testing.assert_close(he.tables.detach(), ref.detach(), rtol=1e-6, atol=1e-7)
