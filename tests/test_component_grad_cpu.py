"""Error paths of the differentiable component modules that need no GPU."""
import pytest
import torch

from nersemble_b200.plugin.components import (HashEnsemble, HashEnsembleConfig, SE3DeformationField,
                                              SE3DeformationFieldConfig, TCNNHashEncodingConfig)


def test_compute_offsets_rejects_position_gradients_before_any_device_call():
    de = SE3DeformationField(torch.tensor([[-1.0, -1, -1], [1, 1, 1]]), SE3DeformationFieldConfig(warp_code_dim=128))
    pos = torch.zeros(4, 3, requires_grad=True)
    with pytest.raises(NotImplementedError, match="positions"):
        de.compute_offsets(pos, torch.zeros(4, 128))
    with torch.no_grad():       # without autograd the same call reaches the (CUDA-only) forward
        with pytest.raises(RuntimeError, match="CUDA|libnsb"):
            de.compute_offsets(pos, torch.zeros(4, 128))


def test_cpu_tensors_that_require_grad_raise_the_cuda_error():
    he = HashEnsemble(HashEnsembleConfig(32, TCNNHashEncodingConfig(log2_hashmap_size=4)))
    assert he.tables.requires_grad
    with pytest.raises(RuntimeError, match="CUDA|libnsb"):
        he(torch.rand(4, 3), torch.rand(4, 32, requires_grad=True))
