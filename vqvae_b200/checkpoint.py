"""Checkpoint interchange with the reference (SURVEY 8f rank 2).

The reference saves ``{'model': state_dict, 'results': {...}, 'hyperparameters': vars(args)}`` with ``torch.save``
(utils.py:106-115, called from main.py:90-93) and loads it in the notebook's ``load_model`` (visualization.ipynb cell 1):
``VQVAE(params['n_hiddens'], params['n_residual_hiddens'], params['n_residual_layers'], params['n_embeddings'],
params['embedding_dim'], params['beta'])`` followed by ``load_state_dict(data['model'])``.  ``load_checkpoint`` does
the same with the drop-in model and packs every conv weight into its kernel layouts right away (not at the first forward).
"""
import torch

from .modules import VQVAE

_HP_KEYS = ("n_hiddens", "n_residual_hiddens", "n_residual_layers", "n_embeddings", "embedding_dim", "beta")


def load_checkpoint(path, device="cuda"):
    """(model, data) from a reference ``.pth``; ``data`` is the loaded dict (``results`` and ``hyperparameters`` untouched)."""
    # the file holds python lists / numpy scalars next to the tensors (main.py:59-64, 81-84): not a weights-only pickle
    data = torch.load(path, map_location="cpu", weights_only=False)
    for k in ("model", "hyperparameters"):
        if k not in data:
            raise KeyError(f"{path}: not a reference checkpoint (missing {k!r}; expected the dict of utils.py:106-115)")
    hp = data["hyperparameters"]
    missing = [k for k in _HP_KEYS if k not in hp]
    if missing:
        raise KeyError(f"{path}: hyperparameters lack {missing}")
    ema = data.get("vq_ema")
    kw = {} if ema is None else dict(ema_decay=ema["decay"], ema_eps=ema["eps"])
    model = VQVAE(hp["n_hiddens"], hp["n_residual_hiddens"], hp["n_residual_layers"], hp["n_embeddings"],
                  hp["embedding_dim"], hp["beta"], **kw)
    model.load_state_dict(data["model"])          # 23 keys incl. the aliased stack.1.* (SURVEY Q1)
    if ema is not None:                           # the EMA buffers travel beside "model" (save_checkpoint)
        vq = model.vector_quantization
        with torch.no_grad():
            vq.ema_cluster_size.copy_(ema["cluster_size"])
            vq.ema_embed_sum.copy_(ema["embed_sum"])
        vq.dead_code_threshold = ema.get("dead_code_threshold")
    model = model.to(device).eval()
    if torch.device(device).type == "cuda":
        with torch.cuda.device(torch.device(device)):
            model.repack()                        # conv weights -> kernel layouts now
    return model, data


def save_checkpoint(model, results, hyperparameters, path):
    """Write the reference's checkpoint format (utils.py:106-115) so its notebook / load_model can read the file.
    A model with an EMA codebook (``ema_decay``) keeps ``model`` to the reference's keys, so that ``load_model`` still
    loads it strictly, and adds ``"vq_ema": {decay, eps, cluster_size, embed_sum}``, plus ``dead_code_threshold`` when
    restarts are on; load_checkpoint rebuilds the EMA model from it."""
    sd = model.state_dict()
    data = {"model": sd, "results": results, "hyperparameters": hyperparameters}
    vq = model.vector_quantization
    if vq.decay is not None:
        prefix = "vector_quantization."
        for k in vq._EMA_KEYS:
            del sd[prefix + k]
        data["vq_ema"] = {"decay": vq.decay, "eps": vq.eps, "cluster_size": vq.ema_cluster_size.detach().cpu(),
                          "embed_sum": vq.ema_embed_sum.detach().cpu()}
        if vq.dead_code_threshold is not None:
            data["vq_ema"]["dead_code_threshold"] = vq.dead_code_threshold
    torch.save(data, path)
