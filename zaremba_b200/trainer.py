"""Fused train / eval step around `Model`: one library call per iteration of
main.py:109-117 (zero_grad, detach, forward, nll_loss, backward, clip_grad_norm_, SGD) and
of main.py:91-94 (perplexity's inner step), plus the data-parallel gradient all-reduce.

Semantics are the reference's: the loss is summed over the batch and averaged over time
(main.py:82-84), so data-parallel ranks SUM their gradients (one `all_reduce` of the flat
gradient buffer) before every rank clips on the global norm and applies the same update --
identical to a single process at `--batch_size B * world_size`.
"""
from __future__ import annotations

import ctypes as C
import math
import os

import numpy as np
import torch
import torch.distributed as dist

from . import _lib
from .parallel import allreduce_sum_
from .model import Model


def minibatch(data, batch_size, seq_length):
    """main.py:61-74: token column -> list of (x, y) [T,B] int64 CPU views (same windows,
    same non-contiguous layout the reference hands to the model)."""
    data = torch.as_tensor(np.asarray(data), dtype=torch.int64).reshape(-1)
    num_batches = data.size(0) // batch_size
    data = data[: num_batches * batch_size].view(batch_size, -1)
    out = []
    width = data.size(1)
    for i in range(0, width - 1, seq_length):
        seqlen = min(seq_length, width - 1 - i)
        if seqlen < width - 1 - i:
            out.append((data[:, i:i + seqlen].transpose(1, 0), data[:, i + 1:i + seqlen + 1].transpose(1, 0)))
    return out


class _NullCtx:
    def __enter__(self):
        return None

    def __exit__(self, *a):
        return False


class _SideStream:
    """`with` block that runs on `side`, ordered after everything already on `cur`; `cur` then waits for it."""

    def __init__(self, cur, side):
        self.cur, self.side = cur, side
        self.ctx = torch.cuda.stream(side)

    def __enter__(self):
        self.side.wait_stream(self.cur)
        self.ctx.__enter__()

    def __exit__(self, *a):
        self.ctx.__exit__(*a)
        self.cur.wait_stream(self.side)
        return False


class Trainer:
    def __init__(self, model: Model, batch_size: int, seq_length: int, process_group=None,
                 keep_clipped_grads: bool = False, data_parallel: bool = True, lazy_update: bool = False):
        """lazy_update: let the SGD update of the upper layers' matrices and of fc.W (HBM-bound, no consumer until the
        next forward reaches them) run beside the NEXT step's forward recurrence kernels instead of at the end of this
        step (zrb_set_lazy_update).  Same arithmetic; every Trainer entry point that reads parameters applies what is
        pending first.  Only YOUR OWN reads or writes of the parameter tensors between two steps need `trainer.flush()`
        before them (state_dict(), checkpoints, .cpu(), load_state_dict): until then `rnns.l>=1.weight_*` and `fc.W` hold
        the previous values.
        data_parallel: when torch.distributed is initialised, shard the batch over the ranks and all-reduce the
        gradients (default).  False = this process trains / evaluates its own replica alone (the sharded ensemble of
        BASELINE configs[4]: one model per GPU, no gradient exchange).
        keep_clipped_grads: after a step `.grad` holds coef * g as clip_grad_norm_ (main.py:115) leaves it.  The
        default skips that store (the values are dead: the next step overwrites them) and `.grad` keeps the raw
        gradients of the step; weights, loss and norm are the same either way."""
        if model.lstm_type != "pytorch":
            raise ValueError("Trainer drives the --lstm_type pytorch layout")
        dev = model.embed.W.device
        if dev.type != "cuda":
            raise RuntimeError("Trainer needs the model on a CUDA device (no CPU fallback)")
        self.model, self.B, self.T, self.dev = model, batch_size, seq_length, dev
        self.pg = process_group
        self._keep_clipped = bool(keep_clipped_grads)
        self._lazy = bool(lazy_update) and model.engine == "tc"
        self._pending = False          # lazy mode: a train step has run since the last flush
        self.world = (dist.get_world_size(process_group)
                      if data_parallel and dist.is_available() and dist.is_initialized() else 1)
        params = model.ordered_parameters()
        # flat layout: the library's order, except that a tied E sits next to fc.b, so that the bucket the projection
        # backward completes (E's G_proj part, fc.b) is one range
        layout = params[1:-1] + [params[0], params[-1]] if model.tied else params
        sizes = [p.numel() for p in layout]
        # one flat parameter buffer and one flat gradient buffer; the nn.Parameters become views
        self.flat_p = torch.empty(sum(sizes), device=dev, dtype=torch.float32)
        # DP transport: "ce" = copy engines over NVLink peer memory (dp_ce.cu, overlaps with backward),
        # "nccl" = one torch.distributed all_reduce after backward.  Default: ce up to 4 ranks, NCCL at 8, where the
        # copy engines need seven small peer copies per phase (not measured on H100 systems)
        # (A third transport -- bucket all-reduces on a few-CTA NCCL communicator, each held back with
        # cuStreamWaitValue32 until the backward recurrence beside it is resident -- was built and HUNG on 2 GPUs: a
        # stream blocked on a value that a kernel queued later on another stream will write can share a hardware work
        # queue with that stream.  Removed.)
        default = "ce" if self.world <= 4 else "nccl"
        self.transport = os.environ.get("ZRB_DP_TRANSPORT", default) if self.world > 1 else None
        if self.transport not in (None, "ce", "nccl"):
            raise ValueError(f"unknown ZRB_DP_TRANSPORT {self.transport!r}")
        self._dp = None
        if self.transport == "ce" and not self._ce_supported():
            self.transport = "nccl"        # multi-node run or no P2P between the GPUs: one NCCL all-reduce instead
        if self.transport == "ce":
            self.flat_g = self._create_ce_transport(sum(sizes))
        else:
            self.flat_g = torch.zeros(sum(sizes), device=dev, dtype=torch.float32)
        off = 0
        with torch.no_grad():
            for p, n in zip(layout, sizes):
                view = self.flat_p[off:off + n].view_as(p)
                view.copy_(p)
                p.data = view
                p.grad = self.flat_g[off:off + n].view_as(p)
                off += n
        self._ps, self._keep_p = model._params_struct(params)
        self._gs, self._keep_g = model._params_struct([p.grad for p in params])
        self.states = model.state_init(batch_size)
        self._st, self._keep_s = model._states_struct(self.states)
        self.loss = torch.zeros((), device=dev)
        self.norm = torch.zeros((), device=dev)
        self.tgt_prob = torch.zeros(batch_size * seq_length, device=dev)
        self._hx = torch.empty(seq_length, batch_size, dtype=torch.int64).pin_memory()
        self._hy = torch.empty(seq_length, batch_size, dtype=torch.int64).pin_memory()
        self._hloss = torch.zeros(2, dtype=torch.float32).pin_memory()
        self.step = 0
        # Dropout keep-flags are Philox(seed, step, site, element).  Data-parallel ranks hold different rows of the
        # global batch, so each rank needs its own stream of flags (identical weights, which bench.py / train_ptb.py
        # get from a common torch seed, must not imply identical masks): the rank is folded into the key.
        rank = dist.get_rank(process_group) if self.world > 1 else 0
        self.seed = (int(torch.initial_seed()) + rank * 0x9E3779B97F4A7C15) & 0xFFFFFFFFFFFFFFFF
        # data-parallel buckets of the flat gradient buffer, in the order backward completes them:
        # [fc.W, fc.b], layer L-1, ..., layer 1, [embed.W + layer 0]
        # (tied: [E, fc.b], layer L-1, ..., layer 1, [layer 0]; E's embedding part travels as rows, added afterwards)
        L = model.layer_num
        offs = [0]
        for n in sizes:
            offs.append(offs[-1] + n)
        r0 = 0 if model.tied else 1            # where layer 0 starts in the flat layout
        self._buckets = [(offs[4 * L], offs[-1])] if model.tied else [(offs[1 + 4 * L], offs[-1])]
        for l in range(L - 1, 0, -1):
            self._buckets.append((offs[r0 + 4 * l], offs[r0 + 4 * (l + 1)]))
        self._buckets.append((0, offs[r0 + 4]))
        self._embed_end = offs[r0]             # all-reduced with the rest from here (tied: E's projection part too)
        self._comm_stream = torch.cuda.Stream(device=dev) if self.world > 1 else None
        # (reducing finished buckets with NCCL underneath the rest of backward was removed: NCCL's channels evict part
        # of the persistent recurrence grid; the copy-engine transport is the one that overlaps)
        self._ctx_cached = None
        self._step_stream = None
        _ = self.ctx
        # single process: the fused step owns the gradient buffers -> touch only the window's embedding rows and take
        # the matrices' clip norm from the wgrad epilogues (mode 1).  Data parallel with the sparse embedding exchange
        # (both transports): rows-only embedding handling over ALL ranks' tokens (mode 2)
        sparse_on = os.environ.get("ZRB_EMBED_SPARSE", "1") == "1"
        self._embed_sparse = (1 if self.world == 1 else 2) if sparse_on else 0
        _lib.check(_lib.load().zrb_set_embed_sparse(self.ctx, self._embed_sparse))
        _lib.check(_lib.load().zrb_set_keep_clipped_grads(self.ctx, 1 if self._keep_clipped else 0))
        _lib.check(_lib.load().zrb_set_lazy_update(self.ctx, 1 if self._lazy else 0))
        if self.world > 1 and self._embed_sparse == 2:
            H, N = model.hidden_size, batch_size * seq_length
            self._rows = torch.zeros(N, H, device=dev)
            self._rows_all = torch.zeros(self.world * N, H, device=dev)
            self._ids_all = torch.zeros(self.world * N, dtype=torch.int64, device=dev)
            # (the rows buffer is handed to the context only for the duration of a DP step, see _grads_ce)

    def _ce_supported(self):
        """The copy-engine transport needs every rank on ONE host (CUDA IPC) with peer access between all GPUs.
        Decided collectively so that all ranks pick the same transport."""
        import socket
        info = [None] * self.world
        dist.all_gather_object(info, (socket.gethostname(), self.dev.index), group=self.pg)
        ok = len({h for h, _ in info}) == 1
        if ok:
            ok = all(i == self.dev.index or torch.cuda.can_device_access_peer(self.dev.index, i) for _, i in info)
        flag = torch.tensor([1 if ok else 0], device=self.dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.pg)
        return bool(flag.item())

    def _create_ce_transport(self, n):
        """zrb_dp_create + CUDA-IPC handle exchange; returns the library-owned flat gradient buffer as a tensor."""
        lib = _lib.load()
        rank = dist.get_rank(self.pg)
        dp = C.c_void_p()
        with torch.cuda.device(self.dev):
            _lib.check(lib.zrb_dp_create(rank, self.world, n, C.byref(dp)))
            blob = (C.c_uint8 * 128)()
            _lib.check(lib.zrb_dp_export(dp, blob))
            mine = torch.tensor(list(blob), dtype=torch.uint8, device=self.dev)
            allb = [torch.empty_like(mine) for _ in range(self.world)]
            dist.all_gather(allb, mine, group=self.pg)
            host = torch.stack(allb).cpu().contiguous()
            _lib.check(lib.zrb_dp_import(dp, C.c_void_p(host.data_ptr())))
        self._dp = dp
        ptr = lib.zrb_dp_grad_buffer(dp)

        class _Ext:       # external CUDA memory -> torch tensor (no ownership), via the CUDA array interface
            __cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (int(ptr), False), "version": 2}

        self._ext = _Ext()
        return torch.as_tensor(self._ext, device=self.dev)

    def _grads_ce(self, lib, x, y, T, B):
        """Backward in phases.  Buckets that finish early (fc, upper layers) are reduced over NVLink by the copy
        engines underneath the rest of backward (zrb_dp_allreduce_bucket: no SM used, so the persistent
        kernels keep the whole chip); the bucket that only completes with the end of backward
        (embed + layer 0) cannot overlap with anything and goes through one NCCL all-reduce."""
        st = self._stream()
        L = self.model.layer_num
        _lib.check(lib.zrb_set_embed_rows_out(self.ctx, _lib.ptr(self._rows)))
        _lib.check(lib.zrb_dp_begin_step(self._dp, st))
        _lib.check(lib.zrb_train_step_begin(self.ctx, C.byref(self._ps), C.byref(self._gs), _lib.ptr(x), _lib.ptr(y),
                                            T, B, C.byref(self._st), C.byref(self._st), self.seed, self.step,
                                            _lib.ptr(self.loss), st))
        nb = len(self._buckets)
        lo, hi = self._buckets[0]
        _lib.check(lib.zrb_dp_allreduce_bucket(self._dp, 0, lo, hi, 0, st))
        k = 1
        for l in range(L - 1, -1, -1):
            _lib.check(lib.zrb_train_step_layer(self.ctx, C.byref(self._ps), C.byref(self._gs), l, st))
            if l >= 1:
                lo, hi = self._buckets[k]
                _lib.check(lib.zrb_dp_allreduce_bucket(self._dp, k, lo, hi, 0, st))
                k += 1
        lo, hi = self._buckets[nb - 1]
        # tail: layer-0 gradients through one NCCL all-reduce (alone on the GPU); the embedding gradient as rows
        allreduce_sum_(self.flat_g[self._embed_end:hi], self.pg)
        if self.model.tied:
            self._ce_join(lib)
        self._exchange_embedding_rows(lib, x, T, B)
        _lib.check(lib.zrb_dp_finish_step(self._dp, st))
        _lib.check(lib.zrb_set_embed_rows_out(self.ctx, None))

    @property
    def ctx(self):
        """The model's library context (re-fetched every call: the model re-creates it when a larger window is
        requested, and a fresh context must be told that the weights are new to it)."""
        c = self.model._context(self.T, self.B)
        if self._ctx_cached is None or c.value != self._ctx_cached:
            _lib.check(_lib.load().zrb_params_changed(c))
            _lib.check(_lib.load().zrb_set_embed_sparse(c, int(getattr(self, "_embed_sparse", 0))))
            _lib.check(_lib.load().zrb_set_keep_clipped_grads(c, 1 if self._keep_clipped else 0))
            _lib.check(_lib.load().zrb_set_lazy_update(c, 1 if getattr(self, "_lazy", False) else 0))
            self._ctx_cached = c.value
        return c

    def flush(self):
        """Apply weight updates deferred by `lazy_update` now (no-op otherwise).  Call before reading parameter tensors
        yourself between steps; train_step / eval_step / perplexity do not need it."""
        _lib.check(_lib.load().zrb_flush_updates(self.ctx, self._stream()))
        self._pending = False

    def params_changed(self):
        """Tell the library that parameter VALUES were changed outside it (model.load_state_dict, a manual edit):
        the fp16 operand images are rebuilt on the next step.  train_step / eval_step also detect in-place writes
        through the tensors' version counters, so calling this is only needed after writes torch cannot see."""
        self.flush()
        _lib.check(_lib.load().zrb_params_changed(self.ctx))
        self._versions = self._param_versions()

    def _param_versions(self):
        return tuple(p._version for p in self.model.parameters())

    def _check_versions(self):
        v = self._param_versions()
        if v != getattr(self, "_versions", None):
            if getattr(self, "_versions", None) is not None and self._lazy and self._pending:
                raise RuntimeError("parameters were modified outside the Trainer while lazy weight updates were still "
                                   "pending: call trainer.flush() before reading or writing parameter tensors")
            _lib.check(_lib.load().zrb_params_changed(self.ctx))
            self._versions = v

    def check_health(self):
        """Raise if a persistent recurrence kernel gave up on a wait (zrb_check_health: one host load, no sync).  Every
        train / eval call checks this on entry anyway; this is for loops that never read anything back."""
        _lib.check(_lib.load().zrb_check_health(self.ctx))

    def close(self):
        """Release the copy-engine transport (IPC mappings, streams)."""
        if getattr(self, "_dp", None) is not None:
            _lib.load().zrb_dp_destroy(self._dp)
            self._dp = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset_states(self):
        for h, c in self.states:
            h.zero_(); c.zero_()

    def _stream(self):
        return torch.cuda.current_stream(self.dev).cuda_stream

    def _own_stream(self):
        """Optional (ZRB_OWN_STREAM=1): when the caller is on the legacy default stream, run the step on a stream of
        the Trainer's own, ordered after the caller's stream and joined back into it afterwards.  Off by default:
        programmatic dependent launches overlap on the legacy default stream as well (tools/micro/pdl_overlap.cu)
        and the two event hops cost ~10 us per step."""
        cur = torch.cuda.current_stream(self.dev)
        if cur.cuda_stream != 0 or os.environ.get("ZRB_OWN_STREAM", "0") != "1":
            return _NullCtx()
        if self._step_stream is None:
            self._step_stream = torch.cuda.Stream(device=self.dev)
        return _SideStream(cur, self._step_stream)

    # ---- main.py:109-117 -----------------------------------------------------------------
    def train_step(self, x, y, lr, max_norm):
        """x, y: [T,B] int64 CUDA tensors (contiguous).  Returns (loss, norm) as 0-d CUDA
        tensors (no host sync)."""
        with self._own_stream():
            return self._train_step(x, y, lr, max_norm)

    def _train_step(self, x, y, lr, max_norm):
        lib = _lib.load()
        T, B = x.shape
        self._check_versions()
        if self.world > 1 and self.transport == "ce":
            self._grads_ce(lib, x, y, T, B)
        else:
            # "nccl": backward in one piece (its weight-gradient GEMMs run beside the recurrence kernels), then ONE
            # all-reduce of everything but the embedding table, whose gradient travels as rows (4 MB per rank
            # instead of 60 MB dense) and is scattered deterministically on every rank
            sparse = self.world > 1 and self._embed_sparse == 2
            if sparse:
                _lib.check(lib.zrb_set_embed_rows_out(self.ctx, _lib.ptr(self._rows)))
            _lib.check(lib.zrb_train_step_grads(self.ctx, C.byref(self._ps), C.byref(self._gs), _lib.ptr(x),
                                                _lib.ptr(y), T, B, C.byref(self._st), C.byref(self._st), self.seed,
                                                self.step, _lib.ptr(self.loss), self._stream()))
            if sparse:
                allreduce_sum_(self.flat_g[self._embed_end:], self.pg)
                self._exchange_embedding_rows(lib, x, T, B)
                _lib.check(lib.zrb_set_embed_rows_out(self.ctx, None))
            elif self.world > 1:
                allreduce_sum_(self.flat_g, self.pg)
        if self._dp is not None and self._keep_clipped:
            # the update rewrites g in place (coef * g) while peers may still be pulling this rank's reduced shards
            # out of it: wait for every peer's "done" flag first (the wait the next step's first write does anyway)
            _lib.check(lib.zrb_dp_begin_step(self._dp, self._stream()))
        _lib.check(lib.zrb_train_step_update(self.ctx, C.byref(self._ps), C.byref(self._gs), float(lr),
                                             float(max_norm), _lib.ptr(self.norm), self._stream()))
        self.step += 1
        self._pending = True
        return self.loss, self.norm

    def _ce_join(self, lib):
        """Tied model on the copy-engine transport: E's gradient lies in bucket 0, which the transport reduces on its
        own streams (peers pull my shard, my shard is reduced in place, the peers' reduced shards are copied in), and
        the scatter (zrb_embed_scatter_rows) then ADDS the embedding rows into that same range in place.  So the add
        must wait until (1) this rank's reduction and gathers of every bucket have finished (zrb_dp_finish_step: the compute stream
        waits for them), and (2) every peer has pulled this rank's reduced shards (zrb_dp_begin_step: the peers' "done"
        flags) -- otherwise a peer could copy a row that already holds e_r and add e_r a second time."""
        st = self._stream()
        _lib.check(lib.zrb_dp_finish_step(self._dp, st))
        _lib.check(lib.zrb_dp_begin_step(self._dp, st))

    def _exchange_embedding_rows(self, lib, x, T, B):
        """Sparse form of the embedding gradient: all-gather every rank's N token ids and N masked gradient rows
        (4 MB per rank instead of a 60 MB dense all-reduce) and scatter them deterministically into the dense buffer."""
        N = T * B
        dist.all_gather_into_tensor(self._rows_all[: self.world * N], self._rows[:N], group=self.pg)
        dist.all_gather_into_tensor(self._ids_all[: self.world * N], x.reshape(-1), group=self.pg)
        _lib.check(lib.zrb_embed_scatter_rows(self.ctx, _lib.ptr(self.model.embed.W.grad), _lib.ptr(self._ids_all),
                                              _lib.ptr(self._rows_all), self.world * N, self._stream()))

    def train_step_host(self, x, y, lr, max_norm):
        """x, y: [T,B] int64 CPU tensors exactly as main.py:71-72 builds them.  Copies them to
        the device, runs the step and returns (loss, norm) as Python floats: the end-to-end
        call (H2D and D2H inside)."""
        lib = _lib.load()
        T, B = x.shape
        hx, hy = self._hx[:T, :B], self._hy[:T, :B]
        if T != self.T or B != self.B:
            hx = torch.empty(T, B, dtype=torch.int64).pin_memory(); hy = torch.empty_like(hx).pin_memory()
        hx.copy_(x); hy.copy_(y)
        if self.world == 1:
            self._check_versions()
            with self._own_stream():
                return self._train_step_host1(lib, hx, hy, T, B, lr, max_norm)
        xd = hx.to(self.dev, non_blocking=True); yd = hy.to(self.dev, non_blocking=True)
        loss, norm = self.train_step(xd, yd, lr, max_norm)
        both = torch.stack([loss, norm]).cpu()
        return float(both[0]), float(both[1])

    def _train_step_host1(self, lib, hx, hy, T, B, lr, max_norm):
        _lib.check(lib.zrb_train_step_host(self.ctx, C.byref(self._ps), C.byref(self._gs),
                                           C.c_void_p(hx.data_ptr()), C.c_void_p(hy.data_ptr()), T, B,
                                           C.byref(self._st), C.byref(self._st), self.seed, self.step,
                                           float(lr), float(max_norm), C.c_void_p(self._hloss.data_ptr()),
                                           C.c_void_p(self._hloss.data_ptr() + 4), self._stream()))
        self.step += 1
        self._pending = True
        return float(self._hloss[0]), float(self._hloss[1])

    # ---- main.py:91-94 --------------------------------------------------------------------
    def eval_step(self, x, y, want_probs=False, cache=None, theta=0.0, lam=0.0):
        """Eval-mode forward + loss on device tokens; carries `self.states`.  Returns the loss
        tensor (main.py:92) and, if asked, softmax(scores)[n, y_n] for the ensemble
        (ensemble.py:100-106).
        cache: a `NeuralCache` -> zrb_eval_step_cache: the window is appended to the cache and the loss is that of
        (1 - lam) p_model + lam p_cache at temperature theta (DESIGN.md section 12).  With want_probs the return is
        (loss, p_model, p_cache), [T*B] each, from which any lam can be evaluated on the host."""
        lib = _lib.load()
        T, B = x.shape
        self._check_versions()
        self._pending = False          # zrb_eval_step applies what is pending before it reads the weights
        if cache is not None:
            return self._eval_step_cache(lib, x, y, T, B, want_probs, cache, theta, lam)
        _lib.check(lib.zrb_eval_step(self.ctx, C.byref(self._ps), _lib.ptr(x), _lib.ptr(y), T, B,
                                     C.byref(self._st), C.byref(self._st), _lib.ptr(self.loss),
                                     _lib.ptr(self.tgt_prob) if want_probs else None, self._stream()))
        return (self.loss, self.tgt_prob[: T * B]) if want_probs else self.loss

    def _eval_step_cache(self, lib, x, y, T, B, want_probs, cache, theta, lam):
        if not hasattr(self, "cache_prob"):
            self.cache_prob = torch.zeros_like(self.tgt_prob)
        _lib.check(lib.zrb_eval_step_cache(self.ctx, C.byref(self._ps), _lib.ptr(x), _lib.ptr(y), T, B,
                                           C.byref(self._st), C.byref(self._st), cache.handle, float(theta), float(lam),
                                           _lib.ptr(self.loss), _lib.ptr(self.tgt_prob) if want_probs else None,
                                           _lib.ptr(self.cache_prob) if want_probs else None, self._stream()))
        if want_probs:
            return self.loss, self.tgt_prob[: T * B], self.cache_prob[: T * B]
        return self.loss

    def perplexity(self, batches, cache=None, theta=0.0, lam=0.0):
        """main.py:86-95 with the per-batch `.item()` sync removed: losses accumulate on the
        device and are read once.  cache: a `NeuralCache`, reset together with the states, through which every window
        is evaluated (eval_step(cache=, theta=, lam=))."""
        self.reset_states()
        if cache is not None:
            cache.reset()
        acc = torch.zeros((), device=self.dev, dtype=torch.float64)
        n = 0
        for x, y in batches:
            xd = x.to(self.dev).contiguous(); yd = y.to(self.dev).contiguous()
            loss = self.eval_step(xd, yd) if cache is None else self.eval_step(xd, yd, cache=cache, theta=theta, lam=lam)
            acc += loss.double() / x.shape[1]
            n += 1
        return math.exp(acc.item() / max(n, 1))

    # ---- dynamic evaluation (DESIGN.md section 14) -------------------------------------------------------------------
    def _single_replica(self, what):
        if self.world > 1:
            raise ValueError(f"{what} adapts one replica: create the Trainer with data_parallel=False")

    def _check_flat(self, flat):
        if flat.shape != self.flat_p.shape or flat.dtype != torch.float32 or flat.device != self.flat_p.device or \
                not flat.is_contiguous():
            raise ValueError(f"expected a contiguous flat fp32 tensor of {self.flat_p.numel()} elements on {self.dev}")

    def _flat_params_struct(self, flat):
        """zrb_params over a flat tensor in flat_p's layout (theta_g, the statistics): views at the parameters' offsets."""
        self._check_flat(flat)
        base = self.flat_p.data_ptr()
        views = [flat[(p.data_ptr() - base) // 4:][:p.numel()].view_as(p) for p in self.model.ordered_parameters()]
        return self.model._params_struct(views)[0]

    def gradient_stats(self, batches):
        """The RMS rule's statistics over `batches` ((x, y) [T,B] windows, one B for all): per window the eval-mode
        gradient at the current weights (no update), states carried from zero; ms += g^2, then r = sqrt(ms / K) and
        r-bar.  The weights are unchanged; pending lazy updates are applied first; the Trainer's states are reset.
        The windows may have another [T,B] than the evaluation ones.  Windows larger than the Trainer's own [T,B] make
        the model re-create its context for the larger shape, and the Trainer then keeps running in that context, whose
        recurrence plans were chosen for the larger batch.  To keep the Trainer's own plans, compute such statistics on
        a Trainer of their shape: a `GradStats` serves every Trainer of the same model configuration (the flat layout
        depends only on the model).  Returns a `GradStats`."""
        from .dyneval import GradStats
        self._single_replica("gradient_stats")
        batches = list(batches)
        if not batches:
            raise ValueError("gradient_stats needs at least one window")
        Bs = {x.shape[1] for x, _ in batches}
        if len(Bs) != 1:
            raise ValueError(f"all statistics windows must have one batch size (got {sorted(Bs)})")
        B = Bs.pop()
        T = max(x.shape[0] for x, _ in batches)
        lib = _lib.load()
        self.flush()
        self._check_versions()
        if T > self.T or B > self.B:     # a larger context for these windows (the Trainer's own still fit in it)
            self.model._context(max(T, self.T), max(B, self.B))
        ctx = self.ctx
        self.reset_states()
        states = self.states if B == self.B else self.model.state_init(B)
        st, keep_s = self.model._states_struct(states)
        ms = torch.zeros_like(self.flat_p)
        ms_s = self._flat_params_struct(ms)
        mean = torch.zeros((), device=self.dev)
        loss = torch.zeros((), device=self.dev)
        for x, y in batches:
            xd = x.to(self.dev).contiguous(); yd = y.to(self.dev).contiguous()
            _lib.check(lib.zrb_grad_stats_step(ctx, C.byref(self._ps), C.byref(self._gs), C.byref(ms_s), _lib.ptr(xd),
                                               _lib.ptr(yd), xd.shape[0], B, C.byref(st), C.byref(st), _lib.ptr(loss),
                                               self._stream()))
        _lib.check(lib.zrb_grad_stats_finish(ctx, C.byref(ms_s), len(batches), _lib.ptr(mean), self._stream()))
        self.reset_states()
        return GradStats(ms, mean, len(batches))

    def dynamic_eval_step(self, x, y, theta_g, lr, lam=0.0, stats=None, eps=2e-5):
        """One window of dynamic evaluation (zrb_dyneval_step): the eval-mode loss at the current weights, then
        theta += a * (theta_g - theta) - lr * u with the RMS rule (stats: a `GradStats`) or the SGD rule (stats None).
        theta_g: flat tensor in flat_p's layout.  Carries `self.states` (so B must not exceed the Trainer's batch);
        returns the 0-d loss tensor (no host sync).  Afterwards `.grad` holds the window's raw gradient."""
        self._single_replica("dynamic_eval_step")
        lib = _lib.load()
        T, B = x.shape
        if B > self.B:
            raise ValueError(f"window batch {B} exceeds the Trainer's batch {self.B} (its states hold {self.B} rows)")
        if stats is not None and (stats.mean.numel() != 1 or stats.mean.dtype != torch.float32
                                  or stats.mean.device != self.flat_p.device):
            raise ValueError(f"stats.mean must be one fp32 element on {self.dev}")
        self._check_flat(theta_g)          # every call; the structs below only hold the pointers
        if stats is not None:
            self._check_flat(stats.rms)
        key = (theta_g.data_ptr(), None if stats is None else stats.rms.data_ptr())
        if getattr(self, "_dyn_key", None) != key:
            self._dyn_structs = (self._flat_params_struct(theta_g),
                                 None if stats is None else self._flat_params_struct(stats.rms))
            self._dyn_key = key
        gl, rms = self._dyn_structs
        self._check_versions()
        self._pending = False          # the call applies what is pending before it reads the weights
        _lib.check(lib.zrb_dyneval_step(self.ctx, C.byref(self._ps), C.byref(self._gs), C.byref(gl),
                                        None if rms is None else C.byref(rms),
                                        None if stats is None else _lib.ptr(stats.mean), _lib.ptr(x), _lib.ptr(y), T, B,
                                        C.byref(self._st), C.byref(self._st), float(lr), float(lam), float(eps),
                                        _lib.ptr(self.loss), self._stream()))
        return self.loss

    def dynamic_perplexity(self, batches, lr, lam=0.0, stats=None, eps=2e-5, restore=True):
        """`perplexity` with dynamic evaluation: applies pending updates, snapshots theta_g = the current weights,
        resets the states, adapts after every window and returns exp(mean over windows of loss / B).  restore: put
        theta_g back afterwards (and tell the library)."""
        self._single_replica("dynamic_perplexity")
        self.flush()
        self._check_versions()
        theta_g = self.flat_p.clone()
        self.reset_states()
        acc = torch.zeros((), device=self.dev, dtype=torch.float64)
        n = 0
        try:
            for x, y in batches:
                xd = x.to(self.dev).contiguous(); yd = y.to(self.dev).contiguous()
                loss = self.dynamic_eval_step(xd, yd, theta_g, lr, lam, stats, eps)
                acc += loss.double() / x.shape[1]
                n += 1
            return math.exp(acc.item() / max(n, 1))
        finally:
            if restore:
                with torch.no_grad():
                    self.flat_p.copy_(theta_g)
                self.params_changed()
