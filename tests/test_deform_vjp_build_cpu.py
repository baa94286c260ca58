"""Build guard for deform_input_grad_kernel (nsb_deform_vjp.cu): it compiles for sm_90a without register spills and inside
the register budget of a 256-thread CTA, and libnsb exports its entry point."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "nersemble_b200", "csrc")
# sinf / sincosf keep their large-argument reduction table on the stack (32 bytes, not a spill); anything above this is
# the compiler moving chain state (ReLU masks, posenc accumulators) to local memory
MAX_SPILL_BYTES = 0
MAX_STACK_BYTES = 64


def test_deform_vjp_kernel_compiles_for_sm90a_without_spills(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("needs nvcc")
    out = subprocess.run([nvcc, "-O3", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-gencode",
                          "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-c", os.path.join(CSRC, "nsb_deform_vjp.cu"),
                          "-o", str(tmp_path / "nsb_deform_vjp.o")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert "warning" not in out.stderr.lower(), out.stderr
    blocks = re.findall(r"Function properties for (\S+)\s+(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads"
                        r"\s+ptxas info\s+: Used (\d+) registers", out.stderr)
    kernels = [b for b in blocks if "deform_input_grad_kernel" in b[0]]
    assert len(kernels) == 1, out.stderr
    _, stack, st, ld, regs = kernels[0]
    assert int(st) <= MAX_SPILL_BYTES and int(ld) <= MAX_SPILL_BYTES and int(stack) <= MAX_STACK_BYTES, kernels[0]
    assert int(regs) <= 255


def test_library_exports_the_entry_point():
    from nersemble_b200 import _lib
    assert "nsb_deform_input_grad" in _lib.SYMBOLS
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as ge
        ge.build()
    assert hasattr(ctypes.CDLL(_lib.LIB_PATH), "nsb_deform_input_grad")
