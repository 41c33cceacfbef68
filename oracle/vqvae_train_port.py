"""The VQ-VAE forward and main.py's loss restated differentiably with torch ops -- TEST INFRASTRUCTURE ONLY.

``vqvae_train_forward`` is the reference's VQVAE.forward (models/vqvae.py:29-44) on a dict of leaf tensors, in fp32 or
fp64, with the quantizer's straight-through estimator and detached loss terms (quantizer.py:63-67).  The argmin has no
gradient, so the indices may be given: an fp64 check of the GPU's gradients is only meaningful at the codes the GPU
chose.  ``train_loss`` is main.py:74-78.  Pinned against the unmodified reference by tests/test_vqvae_train_cpu.py
through the tests/golden/vqvae_grad_* / vqvae_train_* vectors that ``python -m oracle.make_vqvae_grad_golden``
writes.  The product never imports this module.
"""
import torch
import torch.nn.functional as F

from .torch_port import decoder, encoder


def vector_quantizer(z, E, beta, idx=None):
    """quantizer.py:45-76 -> (loss, z_q NCHW, perplexity, idx (N,)); `idx` given: quantize to those codes."""
    z = z.permute(0, 2, 3, 1).contiguous()
    zf = z.view(-1, E.shape[1])
    if idx is None:
        d = torch.sum(zf ** 2, dim=1, keepdim=True) + torch.sum(E ** 2, dim=1) - 2 * torch.matmul(zf, E.t())
        idx = torch.argmin(d, dim=1)
    z_q = E[idx].view(z.shape)                                   # = matmul(one_hot, E), gradient included
    loss = torch.mean((z_q.detach() - z) ** 2) + beta * torch.mean((z_q - z.detach()) ** 2)
    z_q = z + (z_q - z).detach()
    e_mean = torch.bincount(idx, minlength=E.shape[0]).to(z.dtype) / idx.numel()
    perplexity = torch.exp(-torch.sum(e_mean * torch.log(e_mean + 1e-10)))
    return loss, z_q.permute(0, 3, 1, 2).contiguous(), perplexity, idx


def vqvae_train_forward(x, g, n_res, beta=0.25, idx=None):
    """(embedding_loss, x_hat, perplexity, idx) of image x under the parameters g (state-dict keys -> tensors)."""
    z_e = F.conv2d(encoder(x, g, n_res), g["pre_quantization_conv.weight"], g["pre_quantization_conv.bias"])
    loss, z_q, perplexity, idx = vector_quantizer(z_e, g["vector_quantization.embedding.weight"], beta, idx)
    return loss, decoder(z_q, g, n_res), perplexity, idx


def train_loss(x, x_hat, embedding_loss, x_train_var):
    """main.py:75-76 -> (loss, recon_loss)."""
    recon = torch.mean((x_hat - x) ** 2) / x_train_var
    return recon + embedding_loss, recon
