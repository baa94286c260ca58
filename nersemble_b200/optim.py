"""Optimiser for the `fields` parameter group with the hash-table update fused into one CUDA pass.

The reference trains with nerfstudio's AdamOptimizerConfig (torch.optim.Adam, eps = 1e-15) over the 8 dense tcnn grid
gradients (train_nersemble.py: optimizers["fields"]).  For the 403 M-element table that costs, per step, the dense
expansion of the scattered gradient, torch's multi-pass foreach Adam and a fresh fp32 -> fp16 copy
of the table for the next forward.  `FusedFieldsAdam` is a torch.optim.Adam whose update of
the table parameter is nsb_table_adam_step: rank-1 gradient expansion + Adam + fp16 refresh in one streaming pass;
every other parameter of the group goes through torch.optim.Adam unchanged, and the optimiser state keeps torch's
keys (`step`, `exp_avg`, `exp_avg_sq`), so checkpoints interchange with a plain Adam.

    opt = FusedFieldsAdam(model.get_param_groups()["fields"], lr=5e-3, eps=1e-15)     # finds the table by itself

nerfstudio: `FusedFieldsAdamOptimizerConfig` has AdamOptimizerConfig's fields and `setup(params)` signature.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch

from . import ops


class FusedFieldsAdam(torch.optim.Adam):
    """torch.optim.Adam whose update of the HashEnsemble table is one fused CUDA pass.

    GradScaler (engine/nersemble_trainer.py:182-186 runs `grad_scaler.scale(loss).backward(); grad_scaler.step(opt)`):
    the parked rank-1 table gradient is not a `.grad`, so `GradScaler.unscale_` neither unscales nor inf-checks it.
    This class therefore declares `_step_supports_amp_scaling` -- GradScaler.step() then hands `grad_scale` /
    `found_inf` (computed over the `.grad` tensors) to step() instead of deciding itself.  (1) The training backward
    makes a non-finite table-side gradient visible to that check by poisoning the mlp_base gradient with NaN
    (plugin/model.py::_RenderFunction.backward), so the scaler's own found_inf / back-off logic covers it; (2) step()
    skips the WHOLE step when found_inf is set (no inf reaches the 1.6 GB table or its fp16 copy); (3) it unscales both
    the dense `.grad`s and the parked gradient by 1/scale, so the Adam moments are accumulated at the true gradient scale whatever the scaler
    does to its scale.  One host synchronisation (found_inf, scale), where torch's GradScaler.step() has its own.

    DDP: the table's `.grad` is None, so DistributedDataParallel does not reduce it.  step() all-reduces a parked
    gradient that `distributed.allreduce_gradients` has not already reduced whenever a process group with more than
    one rank exists (every rank steps, so every rank issues the collective)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, **kw):
        if kw.get("amsgrad") or kw.get("maximize"):
            raise NotImplementedError("FusedFieldsAdam: amsgrad / maximize")
        super().__init__(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, **kw)
        self._step_supports_amp_scaling = True     # see the class docstring
        # extra factor on the parked gradient for trainers that scale the loss WITHOUT a GradScaler (1 / their scale)
        self.pending_grad_scale = 1.0
        self.auto_allreduce = True
        self.shard_tables = False          # N > 1: reduce-scatter -> Adam on 1/N of the entries -> all-gather of the fp16 table
        self.last_step_skipped = False
        self._ensembles = []
        for group in self.param_groups:
            for p in group["params"]:
                he = getattr(p, "_nsb_hash_ensemble", None)
                he = he() if he is not None else None
                if he is not None:
                    he.defer_table_grad = True     # backward leaves the table gradient in rank-1 form
                    self._ensembles.append((he, p, group))
        if not self._ensembles:
            raise ValueError("FusedFieldsAdam: no HashEnsemble table among the parameters (use torch.optim.Adam)")

    def zero_grad(self, set_to_none: bool = True):
        super().zero_grad(set_to_none)
        for he, _, _ in self._ensembles:
            he.pending_table_grad = None

    # ------------------------------------------------------------------ sharded table optimiser (SURVEY 8e / 8(f)-3)
    @staticmethod
    def _can_shard(he, p) -> bool:
        import torch.distributed as dist
        pend = he.pending_table_grad
        return (pend is not None and not pend.get("reduced") and pend.get("slots_are_timesteps") and p.grad is None
                and p.shape[0] % dist.get_world_size() == 0)

    def _sharded_table_step(self, he, p, st, shadow, pending, gscale, kw) -> None:
        """Reduce-scatter -> Adam on this rank's 1/N of the table entries -> all-gather of the fp16 table.
        The parked gradient [slots][E][2] is reduce-scattered along the ENTRY axis slot by slot (one coalesced NCCL
        group), which leaves [slots][E/N][2] -- exactly the workspace nsb_table_adam_step takes for the contiguous
        entry range [rank E/N, (rank+1) E/N) of the master / moment / fp16 tensors.  Per step and rank: (N-1)/N x 1.2 GB
        reduced + (N-1)/N x 0.8 GB gathered instead of 2 (N-1)/N x 1.2 GB all-reduced, and the 11.7 GB streaming pass of
        the optimiser shrinks to 1/N.  The forward only reads the fp16 table, which is complete on every rank; the fp32
        master and the Adam moments are current on their owner only -- call consolidate() on ALL ranks before a
        state_dict() / checkpoint."""
        import torch.distributed as dist
        world, rank = dist.get_world_size(), dist.get_rank()
        E = p.shape[0]
        n = E // world
        lo = rank * n
        g = pending["g_rank1"]
        T = int(g.shape[0])
        out = torch.empty((T, n, 2), dtype=g.dtype, device=g.device)
        if g.is_cuda:
            with dist._coalescing_manager(device=g.device, async_ops=False):
                for t in range(T):
                    dist.reduce_scatter_tensor(out[t], g[t], op=dist.ReduceOp.SUM)
        else:                                            # gloo (CPU tests of this logic) has no reduce_scatter
            dist.all_reduce(g, op=dist.ReduceOp.SUM)
            out.copy_(g[:, lo:lo + n])
        local = {"g_rank1": out, "cw_slots": pending["cw_slots"], "n_slots": T}
        ops.table_adam_step(p.data[lo:lo + n], st["exp_avg"][lo:lo + n], st["exp_avg_sq"][lo:lo + n], shadow[lo:lo + n],
                            pending=local, grad_scale=gscale / world, **kw)
        mine = shadow[lo:lo + n].clone()                 # 1/N of 0.8 GB: all_gather_into_tensor wants a separate input
        dist.all_gather_into_tensor(shadow.view(-1), mine.view(-1))
        self._sharded = True

    @torch.no_grad()
    def consolidate(self) -> None:
        """All ranks: gather the owners' fp32 master entries and Adam moments so that every replica (and a checkpoint
        written by rank 0) holds the full, current tensors.  No-op unless the sharded table step ran."""
        import torch.distributed as dist
        if not getattr(self, "_sharded", False) or not (dist.is_available() and dist.is_initialized()):
            return
        world, rank = dist.get_world_size(), dist.get_rank()
        for he, p, _ in self._ensembles:
            st = self.state.get(p, {})
            n = p.shape[0] // world
            for t in (p.data, st.get("exp_avg"), st.get("exp_avg_sq")):
                if t is not None:
                    dist.all_gather_into_tensor(t.view(-1), t[rank * n:(rank + 1) * n].clone().view(-1))
        self._sharded = False

    def _amp_state(self):
        """(skip, inv_scale) from the attributes GradScaler.step() sets on optimisers that support amp scaling."""
        gs, fi = getattr(self, "grad_scale", None), getattr(self, "found_inf", None)
        if gs is None and fi is None:
            return False, 1.0
        dev = (gs if gs is not None else fi).device
        # found_inf covers the parked table gradient too: the training backward poisons the mlp_base gradient (a real
        # `.grad` of this optimiser) with NaN whenever the table-side gradient is non-finite (plugin/model.py)
        bad = torch.zeros((), device=dev) if fi is None else fi.detach().float().reshape(-1).sum()
        scale = torch.ones((), device=dev) if gs is None else gs.detach().float().reshape(())
        bad_v, scale_v = torch.stack([bad, scale]).tolist()      # the one host synchronisation of an amp step
        return bad_v > 0, (1.0 / scale_v if gs is not None else 1.0)

    @torch.no_grad()
    def step(self, closure=None):
        import torch.distributed as dist
        multi = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
        sharded = set()
        if multi:
            from .distributed import allreduce_pending
            for he, p, _ in self._ensembles:
                if self.shard_tables and self._can_shard(he, p):
                    sharded.add(id(p))                   # reduced inside the sharded step below
                elif self.auto_allreduce:
                    allreduce_pending(he, average=True)  # also waits for an overlapped reduction
        skip, inv_scale = self._amp_state()
        self.last_step_skipped = skip
        if skip:
            for he, _, _ in self._ensembles:
                he.pending_table_grad = None
            return None
        if inv_scale != 1.0:
            for group in self.param_groups:
                for p in group["params"]:
                    if p.grad is not None:
                        p.grad.mul_(inv_scale)
        work = []
        for he, p, group in self._ensembles:
            if p.grad is not None and he.pending_table_grad is not None:
                # a dense .grad AND a parked rank-1 gradient (second backward before step()): they may carry different
                # scale factors (all-reduce averaging), so fold the parked one into the dense tensor first
                he.materialize_pending(scale=float(self.pending_grad_scale) * inv_scale)
            work.append((he, p, group, p.grad, he.pending_table_grad))
            p.grad = None                   # torch's Adam skips parameters without .grad
        # torch's non-fused Adam asserts that it was not handed amp state: hide it for the inner call
        amp_attrs = {k: getattr(self, k) for k in ("grad_scale", "found_inf") if hasattr(self, k)}
        for k in amp_attrs:
            setattr(self, k, None)
        try:
            loss = super().step(closure)
        finally:
            for k, v in amp_attrs.items():
                setattr(self, k, v)
        for he, p, group, dense, pending in work:
            if dense is None and pending is None:
                continue
            st = self.state[p]
            if len(st) == 0:
                st["step"] = torch.tensor(0.0)
                st["exp_avg"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
            st["step"] += 1
            shadow = he.shadow_buffer()
            gscale = 1.0 if pending is None else float(pending.get("scale", 1.0)) * float(self.pending_grad_scale) * inv_scale
            kw = dict(step=int(st["step"].item()), lr=float(group["lr"]), betas=group["betas"], eps=group["eps"],
                      weight_decay=group["weight_decay"])
            if id(p) in sharded:
                self._sharded_table_step(he, p, st, shadow, pending, gscale, kw)
            else:
                ops.table_adam_step(p.data, st["exp_avg"], st["exp_avg_sq"], shadow, grad=dense, pending=pending, grad_scale=gscale, **kw)
            torch.autograd.graph.increment_version(p)
            torch.autograd.graph.increment_version(shadow)      # written in place by the kernel: caches keyed on the fp16
            he.set_native_tables(shadow)                        # copy's version (NativeParams.frame_table) must see it
            he.pending_table_grad = None
        return loss


@dataclass
class FusedFieldsAdamOptimizerConfig:
    """Drop-in for nerfstudio.engine.optimizers.AdamOptimizerConfig in the method config's `fields` entry."""
    lr: float = 5e-3
    eps: float = 1e-15
    max_norm: Optional[float] = None
    weight_decay: float = 0.0

    def setup(self, params) -> FusedFieldsAdam:
        return FusedFieldsAdam(params, lr=self.lr, eps=self.eps, weight_decay=self.weight_decay)
