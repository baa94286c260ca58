"""Build-output guards for the wgmma tensor role (nsb_field_tensor_role_tc.inc)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_tc_kernels_do_not_serialise_wgmma():
    """Performance guard: when ptxas cannot prove that a warpgroup reaches its wgmma.mma_async instructions converged, it
    waits for each MMA of the deformation chain before issuing the next (info C7520), which made the deformation the
    bound of the render kernels.  Reads the ptxas log that the Makefile writes next to nsb_field.o."""
    log = os.path.join(ROOT, "nersemble_b200", "csrc", "nsb_field.o.ptxas.log")
    if not os.path.exists(log):
        pytest.skip("needs the in-tree ptxas log (make -C nersemble_b200/csrc)")
    text = open(log).read()
    compiled = set(re.findall(r"Compiling entry function '(\w*_tc\w*)'", text))
    assert len(compiled) >= 12, "expected the field_kernel_tc / render_kernel_tc instantiations in the log"
    serialised = sorted(set(re.findall(r"wgmma\.mma_async instructions are serialized.*?function '(\w+)'", text)))
    assert not serialised, serialised
