"""Spill guard for the wgmma inference kernels (field_kernel_tc / render_kernel_tc).  The deformation chain keeps each
layer's activations in registers (A operand 32 + accumulator 32 + the first half of the next A operand 16 per thread)
inside the tensor role's setmaxnreg budget, so a change that adds state carried across the chain shows up as local-memory
traffic.  Counts STL / LDL per warp-role region of the SASS, with the rule of tools/spill_report.py: the gather region
starts at USETMAXREG.DEALLOC, the tensor region at USETMAXREG.TRY_ALLOC."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "nersemble_b200", "csrc", "nsb_field.o")

TENSOR_MAX = 5      # the tensor role's spill instructions before the chain moved into registers (all 12 kernels)
# gather-role spill instructions per kernel; the gather code is not part of the chain, so any change here means ptxas
# re-allocated the whole kernel around the tensor role
GATHER = {
    "render_kernel_tcILi2ELb1ELb0E": 0, "render_kernel_tcILi2ELb1ELb1E": 0, "render_kernel_tcILi2ELb0ELb0E": 2,
    "render_kernel_tcILi4ELb1ELb0E": 0, "render_kernel_tcILi4ELb1ELb1E": 0, "render_kernel_tcILi4ELb0ELb0E": 2,
    "field_kernel_tcILb1ELb1ELb0E": 0, "field_kernel_tcILb1ELb1ELb1E": 0, "field_kernel_tcILb1ELb0ELb0E": 0,
    "field_kernel_tcILb0ELb1ELb0E": 0, "field_kernel_tcILb0ELb1ELb1E": 0, "field_kernel_tcILb0ELb0ELb0E": 0,
}


def _region_spills(obj):
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    rows, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            rows[cur] = {"region": "pre", "pre": 0, "gather": 0, "tensor": 0}
            continue
        if cur is None:
            continue
        r = rows[cur]
        if "USETMAXREG.DEALLOC" in line:
            r["region"] = "gather"
        elif "USETMAXREG.TRY_ALLOC" in line:
            r["region"] = "tensor"
        if re.search(r"\b(STL|LDL)\b|\bSTL\.|\bLDL\.", line):
            r[r["region"]] += 1
    return rows


def test_tc_kernels_spill_no_more_than_before():
    if not os.path.exists(OBJ):
        pytest.skip("needs the in-tree object (make -C nersemble_b200/csrc)")
    rows = _region_spills(OBJ)
    found = {}
    for key, want_gather in GATHER.items():
        names = [k for k in rows if key in k]
        assert len(names) == 1, (key, names)
        found[key] = rows[names[0]]
    bad = {k: (r["tensor"], r["gather"]) for k, r in found.items()
           if r["tensor"] > TENSOR_MAX or r["gather"] != GATHER[k] or r["pre"] != 0}
    assert not bad, f"(tensor, gather) spill instructions: {bad}"
