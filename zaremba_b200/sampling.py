"""On-device sampling from a score matrix: `sample(scores, ...)` draws one token per row through zrb_sample, and
`beam_step(scores, ...)` runs one selection step of a beam search through zrb_beam_step.

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


def beam_step(scores, beams, cum=None, last_tokens=None, eos=None):
    """One beam-search selection step over the rows of `scores` ([B*K_in, V] fp32 CUDA tensor, finite).

    cum None is the first step: one row per prompt, cumulative score 0, no last token.  Otherwise row b*K + i is slot i
    of prompt b (K = `beams`), with cumulative score cum[row] and last token last_tokens[row] (None: no row is finished);
    a row whose last token is `eos` only extends with eos at log-probability 0.  The `beams` best candidates of each
    prompt -- S + logp descending, ties by the lower slot * V + token -- become its new slots in that order (DESIGN.md
    section 10).
    Returns (tokens int64, parents int32, cum fp32, logprobs fp32), each [B*beams].  No host synchronisation.
    """
    if not scores.is_cuda or scores.dtype != torch.float32 or scores.dim() != 2:
        raise TypeError("beam_step() takes a [rows, V] fp32 CUDA tensor")
    if scores.stride(1) != 1 or scores.stride(0) < scores.size(1):
        scores = scores.contiguous()
    R, V = scores.shape
    K = int(beams)
    if cum is None and last_tokens is not None:
        raise ValueError("the first step (cum None) has no last tokens")
    K_in = 1 if cum is None else K
    if R % K_in:
        raise ValueError(f"{R} rows are not a whole number of prompts of {K_in} slots")
    B = R // K_in
    dev = scores.device
    if cum is not None:
        cum = cum.to(device=dev, dtype=torch.float32).contiguous()
    if last_tokens is not None:
        last_tokens = last_tokens.to(device=dev, dtype=torch.int64).contiguous()
    tokens = torch.empty(B * K, dtype=torch.int64, device=dev)
    parents = torch.empty(B * K, dtype=torch.int32, device=dev)
    cum_out = torch.empty(B * K, dtype=torch.float32, device=dev)
    logprobs = torch.empty(B * K, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.load().zrb_beam_step(_lib.ptr(scores), scores.stride(0), B, K_in, K, V, _lib.ptr(cum),
                                             _lib.ptr(last_tokens), -1 if eos is None else int(eos), _lib.ptr(tokens),
                                             _lib.ptr(parents), _lib.ptr(cum_out), _lib.ptr(logprobs),
                                             torch.cuda.current_stream(dev).cuda_stream))
    return tokens, parents, cum_out, logprobs
