"""Batch-sharded VQVAE.forward on 2 GPUs (NCCL) equals the single-process forward on the concatenated
batch (SURVEY 8e).  Needs >= 2 H100s; skipped on a machine with one GPU."""
import os
import socket

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out_dir):
    import torch.distributed as dist
    from vqvae_b200.synth import make_images, make_state_dict
    from tests.helpers import build_model
    from vqvae_b200.dist import shard_bounds
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    hp = dict(h_dim=128, res_h_dim=32, n_res_layers=2, n_embeddings=512, embedding_dim=64)
    sd = make_state_dict(seed=0, codebook="normal", codebook_scale=0.05, **hp)
    m = build_model(hp, sd, device=f"cuda:{rank}")
    x = make_images(64, 32, seed=1)
    lo, hi = shard_bounds(64, rank, world)
    m.process_group = dist.group.WORLD
    loss, x_hat, perp = m(torch.from_numpy(x[lo:hi]).cuda())
    idx = m.last_min_encoding_indices
    torch.cuda.synchronize()
    # lazy scalars: no collective inside the forward, whole-batch values on demand
    m.sync_scalars = False
    loss_l, x_hat_l, perp_l = m(torch.from_numpy(x[lo:hi]).cuda())
    loss_r, perp_r = m.reduce_scalars()
    m.sync_scalars = True
    torch.cuda.synchronize()
    np.savez(os.path.join(out_dir, f"r{rank}.npz"), loss=loss.cpu().numpy(), perp=perp.cpu().numpy(),
             x_hat=x_hat.cpu().numpy(), idx=idx.cpu().numpy(), loss_local=loss_l.cpu().numpy(), perp_local=perp_l.cpu().numpy(),
             loss_reduced=loss_r.cpu().numpy(), perp_reduced=perp_r.cpu().numpy(), x_hat_lazy=x_hat_l.cpu().numpy())
    if rank == 0:
        m.process_group = None
        loss1, x_hat1, perp1 = m(torch.from_numpy(x).cuda())
        np.savez(os.path.join(out_dir, "single.npz"), loss=loss1.cpu().numpy(), perp=perp1.cpu().numpy(),
                 x_hat=x_hat1.cpu().numpy(), idx=m.last_min_encoding_indices.cpu().numpy())
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_shards_equal_single_process(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    r0, r1, one = (np.load(tmp_path / f) for f in ("r0.npz", "r1.npz", "single.npz"))
    # sharded tensors, concatenated rank-major, are bitwise the single-process ones
    assert np.array_equal(np.concatenate([r0["x_hat"], r1["x_hat"]]), one["x_hat"])
    assert np.array_equal(np.concatenate([r0["idx"], r1["idx"]]), one["idx"])
    # the two cross-sample scalars agree on every rank and with the single-process forward
    for r in (r0, r1):
        np.testing.assert_allclose(r["loss"], one["loss"], rtol=1e-6)
        np.testing.assert_allclose(r["perp"], one["perp"], rtol=1e-6)
        # sync_scalars = False: the forward returns the shard's own scalars (no collective), reduce_scalars() the whole batch's
        np.testing.assert_allclose(r["loss_reduced"], one["loss"], rtol=1e-6)
        np.testing.assert_allclose(r["perp_reduced"], one["perp"], rtol=1e-6)
        assert np.array_equal(r["x_hat_lazy"], r["x_hat"])
    np.testing.assert_allclose(0.5 * (r0["loss_local"] + r1["loss_local"]), one["loss"], rtol=1e-6)   # equal shards: the mean of means
    assert not np.allclose(r0["perp_local"], r1["perp_local"], rtol=1e-9)                            # really per-shard values
