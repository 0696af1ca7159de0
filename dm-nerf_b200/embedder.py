"""Positional encoder with the reference's interface (networks/dm_nerf.py:8-55): `get_embedder(multires, i)`
returns `(embedder, out_dim)`; `embedder.embed(x)` maps [...,3] -> [..., 3 + 6*multires]."""
import torch
import torch.nn as nn

from . import _lib
from .engine import get_context


class Embedder:
    def __init__(self, **kwargs):
        self.kwargs = kwargs
        if not (kwargs.get("include_input", True) and kwargs.get("log_sampling", True)
                and kwargs.get("input_dims", 3) == 3
                and kwargs.get("max_freq_log2") == kwargs.get("num_freqs", 0) - 1):
            raise NotImplementedError("only the configuration built by get_embedder() is supported "
                                      "(include_input, log_sampling, 3 input dims, sin/cos)")
        self.num_freqs = int(kwargs["num_freqs"])
        self.out_dim = 3 + 6 * self.num_freqs

    def embed(self, inputs):
        if not inputs.is_cuda:
            raise RuntimeError("Embedder.embed: expected a CUDA tensor (no CPU fallback)")
        x = inputs.reshape(-1, 3).contiguous().float()
        out = torch.empty((x.shape[0], self.out_dim), device=x.device, dtype=torch.float32)
        ctx = get_context(x.device)
        ctx.call("dmnerf_posenc", _lib.ptr(x), x.shape[0], self.num_freqs, _lib.ptr(out))
        return out.reshape(*inputs.shape[:-1], self.out_dim)


def get_embedder(multires, i=0):
    if i == -1:
        return nn.Identity(), 3
    embedder = Embedder(include_input=True, input_dims=3, max_freq_log2=multires - 1, num_freqs=multires,
                        log_sampling=True, periodic_fns=[torch.sin, torch.cos])
    return embedder, embedder.out_dim
