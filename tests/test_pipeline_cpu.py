"""Host-side logic of vqvae_b200.HostPipeline that needs no GPU: argument checks and the packed-scalar
detection (the kernels themselves are covered by tests/test_gpu_pipeline.py on an H100)."""
import pytest
import torch


def test_pipeline_refuses_cpu_model():
    import vqvae_b200
    m = vqvae_b200.VQVAE(16, 8, 1, 32, 8, 0.25)              # parameters on the CPU
    with pytest.raises(RuntimeError, match="CUDA"):           # no CPU path exists
        vqvae_b200.HostPipeline(m, (2, 3, 8, 8))


def test_packed_scalars_detection():
    from vqvae_b200.pipeline import _packed_scalars_ptr
    out = torch.zeros(2, dtype=torch.float32)
    assert _packed_scalars_ptr(out[0], out[1]) == out.data_ptr()          # adjacent views of one buffer (ops.vq_finish)
    assert _packed_scalars_ptr(out[1], out[0]) is None                     # wrong order
    assert _packed_scalars_ptr(torch.zeros(()), torch.zeros(())) is None   # unrelated tensors
    assert _packed_scalars_ptr(out[0].double(), out[1]) is None            # wrong dtype


def test_module_forward_refuses_cpu_tensor():
    """models/vqvae.py:29 on a CPU tensor: the product path fails loudly instead of falling back."""
    import vqvae_b200
    m = vqvae_b200.VQVAE(16, 8, 1, 32, 8, 0.25)
    with pytest.raises(RuntimeError):
        m(torch.zeros(1, 3, 8, 8))
