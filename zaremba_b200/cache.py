"""Neural-cache evaluation (Grave, Joulin & Usunier 2017, "Improving Neural Language Models with a Continuous Cache").

    cache = zaremba_b200.NeuralCache(hidden=650, batch=20, size=2000, max_seq=35)
    ppl = trainer.perplexity(batches, cache=cache, theta=0.3, lam=0.1)

The cache keeps, per stream, the last `size` pairs (last-layer hidden state, next token) and mixes the softmax with
the distribution over recently seen words its attention gives (DESIGN.md section 12; include/zaremba_b200.h).
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib


class NeuralCache:
    """zrb_cache_create: the per-stream ring of (key, token) pairs for `batch` streams of a model of width `hidden`,
    holding the last `size` positions; windows of at most `max_seq` rows.  Independent of any model or context."""

    def __init__(self, hidden: int, batch: int, size: int, max_seq: int, device=None):
        self.hidden, self.batch, self.size, self.max_seq = int(hidden), int(batch), int(size), int(max_seq)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self._h = None
        h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().zrb_cache_create(self.hidden, self.batch, self.size, self.max_seq, C.byref(h)))
        self._h = h

    @property
    def handle(self):
        return self._h

    def reset(self):
        """Forget everything: the next token of every stream starts with an empty cache."""
        _lib.check(_lib.load().zrb_cache_reset(self._h))

    def close(self):
        if getattr(self, "_h", None) is not None:
            _lib.load().zrb_cache_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _check_theta_lam(theta, lam):
    if not (theta >= 0.0 and theta < float("inf")):
        raise ValueError(f"theta must be finite and >= 0 (got {theta})")
    if lam is not None and not (0.0 <= lam < 1.0):
        raise ValueError(f"lam must lie in [0, 1) (got {lam})")


def cache_step(cache: NeuralCache, h: torch.Tensor, y: torch.Tensor, theta: float) -> torch.Tensor:
    """zrb_cache_step: append h [T,B,H] (fp32, rounded to fp16 as keys) and targets y [T,B] to `cache`, return p_cache
    [T*B] of every row (row n = t*B + b) against the positions before it."""
    T, B, H = h.shape
    if H != cache.hidden or tuple(y.shape) != (T, B):
        raise ValueError(f"h {tuple(h.shape)} / y {tuple(y.shape)} do not match the cache (H = {cache.hidden})")
    _check_theta_lam(theta, None)
    h = h.to(cache.device, torch.float32).contiguous()
    y = y.to(cache.device, torch.int64).contiguous()
    out = torch.empty(T * B, device=cache.device)
    with torch.cuda.device(cache.device):
        _lib.check(_lib.load().zrb_cache_step(cache.handle, _lib.ptr(h), _lib.ptr(y), T, B, float(theta), _lib.ptr(out),
                                              torch.cuda.current_stream(cache.device).cuda_stream))
    return out
