"""On-device sampling from a score matrix: `sample(scores, ...)` draws one token per row through zrb_sample.

The draw is Gumbel-max over a kept set (top-k, then top-p over the top-k set), a pure function of
(scores, seed, pos, row): DESIGN.md section 9 states it bit for bit.  `Model.generate` runs the same kernel inside
its decode loop, so `sample` applied to the scores of `Model.forward` replays a generation exactly.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib


def sampling_config(temperature=1.0, top_k=0, top_p=1.0, seed=0):
    """The zrb_sampling struct (the library validates the values)."""
    return _lib.ZrbSampling(float(temperature), int(top_k), float(top_p), 0, int(seed) & 0xFFFFFFFFFFFFFFFF)


def sample(scores, temperature=1.0, top_k=0, top_p=1.0, seed=0, pos=0):
    """One token per row of `scores` ([B,V] or [V] fp32 CUDA tensor, finite).

    temperature 0 is greedy (argmax, lowest index on ties); top_k = 0 and top_p = 1 switch the filters off.
    Returns (tokens int64, logprobs fp32) with the leading shape of `scores` minus V; logprobs is
    log softmax(scores)[token] at temperature 1 over the whole row.  No host synchronisation.
    """
    if not scores.is_cuda or scores.dtype != torch.float32:
        raise TypeError("sample() takes an fp32 CUDA tensor")
    squeeze = scores.dim() == 1
    s2 = scores.view(1, -1) if squeeze else scores
    if s2.dim() != 2:
        raise ValueError(f"scores must be [B,V] or [V], got {tuple(scores.shape)}")
    if s2.stride(1) != 1 or s2.stride(0) < s2.size(1):
        s2 = s2.contiguous()
    B, V = s2.shape
    dev = s2.device
    tokens = torch.empty(B, dtype=torch.int64, device=dev)
    logprobs = torch.empty(B, dtype=torch.float32, device=dev)
    cfg = sampling_config(temperature, top_k, top_p, seed)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().zrb_sample(_lib.ptr(s2), s2.stride(0), B, V, C.byref(cfg), int(pos) & 0xFFFFFFFFFFFFFFFF,
                                          _lib.ptr(tokens), _lib.ptr(logprobs), torch.cuda.current_stream(dev).cuda_stream))
    return (tokens[0], logprobs[0]) if squeeze else (tokens, logprobs)
