import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def load_golden(name):
    import json
    import numpy as np
    import torch
    z = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
    meta = json.loads(bytes(z["meta_json"]).decode())
    t = {k: torch.from_numpy(z[k]) for k in z.files if k != "meta_json"}
    return t, meta


_PARAM_CACHE = {}


def oracle_params(knobs):
    """random_params is deterministic in its knobs; cache (full-size tables take seconds)."""
    from oracle import pipeline as pl
    key = tuple(sorted(knobs.items()))
    if key not in _PARAM_CACHE:
        if len(_PARAM_CACHE) > 2:
            _PARAM_CACHE.clear()
        _PARAM_CACHE[key] = pl.random_params(**knobs)
    return _PARAM_CACHE[key]


def native_from_oracle(P, device="cuda", tcgen05=None):
    """oracle FieldParams -> nersemble_b200.ops.NativeParams (same numbers, kernel layouts)."""
    from nersemble_b200 import ops, packing
    lv = P.levels
    levels = dict(n_levels=lv.n_levels, scale=[float(x) for x in lv.scale], res=[int(x) for x in lv.res],
                  entries=[int(x) for x in lv.entries], offset=[int(x) for x in lv.offset[:-1]],
                  hashed=[int(x) for x in lv.hashed], total_entries=lv.total_entries)
    deform = dict(stem_w=P.deform_w, stem_b=P.deform_b, r_w=P.r_w, r_b=P.r_b, v_w=P.v_w, v_b=P.v_b)
    return ops.NativeParams.build(tables=P.tables, base_w=P.base_w, head_w=P.head_w, time_emb=P.time_emb,
                                  aabb=P.aabb, levels=levels, deform=deform, time_emb_deform=P.time_emb_deform,
                                  device=device, tcgen05=tcgen05)
