"""Float64 references of the hash-grid backward (nsb_field_backward's hash pass), device-agnostic, for batch-scale
checks: plain torch on whatever device the inputs live on, no autograd, no dense float64 member tables.

The kernels' inputs are taken as given (the saved float32 `xs`, the kernel's own `d_feat`, the fp16 table), and every
index / trilinear weight is recomputed exactly as the kernels form it (oracle.tp.tcnn_cpu.hashgrid_indices_weights),
so what is left between a kernel and these references is float32 summation and product rounding only.  Each reference
comes with the float64 sum of the absolute values of its terms and a term count, from which the tests derive their
bounds.  Samples with xs.w == 0 (outside the box) contribute like any other: the forward zeroed their coordinates, not
their weights."""
import torch

from oracle.tp.tcnn_cpu import hashgrid_indices_weights

U32 = 2.0 ** -24          # unit roundoff of float32 round-to-nearest


def cw16(codes: torch.Tensor, cw_scale, cw_bias) -> torch.Tensor:
    """Blend weights as the kernels round them, __float2half_rn(fmaf(code, cw_scale, cw_bias)) (nsb_backward.cu
    hash_bwd_kernel / hash_expand_kernel), as float64.  code * scale is exact in float64 (24 x 24 bits); with a zero
    bias (every window >= 2) the whole fma is, so the float32 rounding below is the fma's one."""
    sc = torch.as_tensor(cw_scale, dtype=torch.float32, device=codes.device).double()
    bi = torch.as_tensor(cw_bias, dtype=torch.float32, device=codes.device).double()
    return (codes.double() * sc + bi).float().half().double()


def frac_weights(xs: torch.Tensor, levels):
    """Per-level fractional positions [n, L, 3] (float32, the kernels' px - floorf(px) with px = fmaf(scale, x, 0.5))."""
    x = xs[:, :3].float()
    out = []
    for l in range(levels.n_levels):
        pos = (x.double() * float(levels.scale[l]) + 0.5).float()
        out.append(pos - torch.floor(pos))
    return torch.stack(out, 1)


def hash_scatter_ref(levels, xs: torch.Tensor, d_feat: torch.Tensor, sample_slot: torch.Tensor, n_slots: int):
    """Per-slot 2-vector table gradient of the hash scatter, G[slot, entry, f] = sum over (sample, level, corner)
    hitting `entry` of w * d_feat[level, f], in float64, with A = the matching sums of |w * d_feat| and
    K[slot, entry] = the number of contributions.  `sample_slot` [n] is the slot of each sample's timestep.
    Returns (G [S,E,2] f64, A [S,E,2] f64, K [S,E] f32, touched [S,E] bool): an entry is touched when some contribution
    is non-zero (the kernels skip exact-zero products: a zero weight or a zero feature gradient)."""
    dev = xs.device
    E = levels.total_entries
    n = xs.shape[0]
    G = torch.zeros((n_slots * E, 2), dtype=torch.float64, device=dev)
    A = torch.zeros_like(G)
    K = torch.zeros((n_slots * E,), dtype=torch.float32, device=dev)
    step = 1 << 15
    for a in range(0, n, step):
        b = min(n, a + step)
        idx, w = hashgrid_indices_weights(xs[a:b, :3].float(), levels)       # [m, L, 8]
        flat = (sample_slot[a:b].long()[:, None, None] * E + idx).reshape(-1)
        g = w.double()[..., None] * d_feat[a:b].double().view(-1, levels.n_levels, 1, 2)
        G.index_add_(0, flat, g.reshape(-1, 2))
        A.index_add_(0, flat, g.abs().reshape(-1, 2))
        K.index_add_(0, flat, torch.ones_like(flat, dtype=torch.float32))
    G, A, K = G.view(n_slots, E, 2), A.view(n_slots, E, 2), K.view(n_slots, E)
    return G, A, K, A.sum(-1) > 0


def dense_table_grad(G, A, K, cw_slots: torch.Tensor, lines: torch.Tensor):
    """Dense table gradient on the given lines: ref[line, m, f] = sum_slots cw16[slot, m] * G[slot, line, f], its
    abs-sum sum_slots |cw16| * A and the line's contribution count sum_slots K (the terms of the kernel's sum)."""
    cw = cw_slots.double()                                    # [S, 32]
    g, a = G[:, lines], A[:, lines]                           # [S, m, 2]
    ref = torch.einsum("sm,sef->emf", cw, g)
    ab = torch.einsum("sm,sef->emf", cw.abs(), a)
    return ref, ab, K[:, lines].sum(0)


def code_grad_from_G(G, tables_half: torch.Tensor, cw_scale, step: int = 1 << 20):
    """Time-code gradient of every slot from the rank-1 form, the way hash_expand_kernel forms it:
    code[slot, m] = cw_scale[m] * sum_e sum_f V[e, m, f] * G[slot, e, f] (float64, in line blocks of `step`)."""
    S, E, _ = G.shape
    out = torch.zeros((S, 32), dtype=torch.float64, device=G.device)
    for a in range(0, E, step):
        b = min(E, a + step)
        out += torch.einsum("emf,sef->sm", tables_half[a:b].double(), G[:, a:b])
    return out * torch.as_tensor(cw_scale, dtype=torch.float32, device=G.device).double()


def per_sample_terms(levels, xs: torch.Tensor, d_feat: torch.Tensor, tables_half: torch.Tensor,
                     cw_rows: torch.Tensor, cw_scale, corner_vals=None):
    """Per-sample time-code gradient and position gradient of the hash blend, float64, with their abs-sums:
      code[s, m] = cw_scale[m] * sum_{l, c, f} V[e(l,c), m, f] * w(l,c) * d_feat[l, f]
      d_xs[s, d] = sum_{l, c} +-scale_l * (d_feat[l] . pb(l,c)) * (product of the two other weight factors)
    where V is the fp16 table, cw_rows [n, 32] the sample's fp16-rounded blend weights and pb the member-blended corner
    value sum_m cw[m] * V[e, m] -- or, with corner_vals [n, L, 8, 2] (the training forward's saved fp16 values), those.
    The d_xs terms are expanded to (level, corner, member, f) for the abs-sum when pb comes from the table.
    Returns code [n,32], code_abs [n,32], d_xs [n,3], d_xs_abs [n,3]; d_xs is multiplied by the selector xs.w."""
    dev = xs.device
    n, L = xs.shape[0], levels.n_levels
    sc32 = torch.as_tensor(cw_scale, dtype=torch.float32, device=dev).double()
    scale = torch.as_tensor(levels.scale, dtype=torch.float32, device=dev).double()
    bits = torch.tensor([[(c >> k) & 1 for k in range(3)] for c in range(8)], device=dev, dtype=torch.bool)   # [8,3]
    code = torch.empty((n, 32), dtype=torch.float64, device=dev); code_abs = torch.empty_like(code)
    dxs = torch.empty((n, 3), dtype=torch.float64, device=dev); dxs_abs = torch.empty_like(dxs)
    step = 1 << 13
    for a in range(0, n, step):
        b = min(n, a + step)
        idx, w = hashgrid_indices_weights(xs[a:b, :3].float(), levels)             # [m, L, 8]
        fr = frac_weights(xs[a:b], levels)                                          # [m, L, 3] float32
        df = d_feat[a:b].double().view(-1, L, 1, 2)                                 # [m, L, 1, 2]
        V = tables_half[idx.reshape(-1)].double().view(b - a, L, 8, 32, 2)          # [m, L, 8, 32, 2]
        cw = cw_rows[a:b].double()[:, None, None, :, None]                          # [m, 1, 1, 32, 1]
        wd = w.double()[..., None, None] * df[:, :, :, None, :]                     # [m, L, 8, 1, 2]
        code[a:b] = (V * wd).sum((1, 2, 4)) * sc32
        code_abs[a:b] = (V * wd).abs().sum((1, 2, 4)) * sc32.abs()
        # weight factors per (level, corner, dim), float32 like the kernels': frac where the corner's bit is set, else 1 - frac
        wf = torch.where(bits[None, None], fr[:, :, None, :], 1.0 - fr[:, :, None, :]).double()   # [m, L, 8, 3]
        other = torch.stack([wf[..., 1] * wf[..., 2], wf[..., 0] * wf[..., 2], wf[..., 0] * wf[..., 1]], -1)
        sign = torch.where(bits, 1.0, -1.0).double()[None, None]                             # [1, 1, 8, 3]
        fac = scale[None, :, None, None] * sign * other                                      # [m, L, 8, 3]
        if corner_vals is None:
            t = (cw * V * df[:, :, :, None, :])                                             # [m, L, 8, 32, 2]
            dxs[a:b] = torch.einsum("mlc,mlcd->md", t.sum((3, 4)), fac)
            dxs_abs[a:b] = torch.einsum("mlc,mlcd->md", t.abs().sum((3, 4)), fac.abs())
        else:
            pb = corner_vals[a:b].double().view(b - a, L, 8, 2)
            t = pb * df                                                                     # [m, L, 8, 2]
            dxs[a:b] = torch.einsum("mlc,mlcd->md", t.sum(-1), fac)
            dxs_abs[a:b] = torch.einsum("mlc,mlcd->md", t.abs().sum(-1), fac.abs())
        sel = xs[a:b, 3:4].double()
        dxs[a:b] *= sel; dxs_abs[a:b] *= sel
    return code, code_abs, dxs, dxs_abs
