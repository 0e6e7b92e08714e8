"""Fused train / eval step around `Model`: one library call per iteration of
main.py:109-117 (zero_grad, detach, forward, nll_loss, backward, clip_grad_norm_, SGD) and
of main.py:91-94 (perplexity's inner step), plus the data-parallel gradient all-reduce.

Semantics are the reference's: the loss is summed over the batch and averaged over time
(main.py:82-84), so data-parallel ranks SUM their gradients (one `all_reduce` of the flat
gradient buffer) before every rank clips on the global norm and applies the same update --
identical to a single process at `--batch_size B * world_size`.
"""
from __future__ import annotations

import contextlib
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


def _adam_hyper(betas, eps):
    """(betas, eps) as floats, ValueError outside torch.optim.Adam's domain of the fused rule: 0 <= beta < 1, eps > 0."""
    try:
        b1, b2 = (float(b) for b in betas)
        eps = float(eps)
    except (TypeError, ValueError):
        raise ValueError(f"betas must be two numbers and eps a number, got {betas!r}, {eps!r}") from None
    for name, b in (("beta1", b1), ("beta2", b2)):
        if not (math.isfinite(b) and 0.0 <= b < 1.0):
            raise ValueError(f"{name} must be in [0, 1), got {b!r}")
    if not (math.isfinite(eps) and eps > 0.0):
        raise ValueError(f"eps must be finite and > 0, got {eps!r}")
    return (b1, b2), eps


def adam_state_to_torch(flat_m, flat_v, step, layout, lr, betas, eps):
    """torch.optim.Adam's state_dict() from flat moments: layout = [(state index, shape, offset into the flat
    buffers)].  Per index `step` (a float tensor, as torch keeps it), `exp_avg` and `exp_avg_sq` (copies); no state
    before the first step, as a fresh torch.optim.Adam has none."""
    state = {}
    if step > 0:
        for i, shape, off in layout:
            n = math.prod(shape)
            state[i] = {"step": torch.tensor(float(step)), "exp_avg": flat_m[off:off + n].view(shape).clone(),
                        "exp_avg_sq": flat_v[off:off + n].view(shape).clone()}
    group = {"lr": float(lr), "betas": tuple(betas), "eps": float(eps), "weight_decay": 0, "amsgrad": False,
             "maximize": False, "foreach": None, "capturable": False, "differentiable": False, "fused": None,
             "decoupled_weight_decay": False, "params": [i for i, _, _ in layout]}
    return {"state": state, "param_groups": [group]}


def adam_state_from_torch(sd, layout, flat_m, flat_v):
    """The inverse of adam_state_to_torch: copies the moments into flat_m / flat_v (zeros for an empty state) and
    returns (step, betas, eps, lr).  ValueError unless sd has one param group over the layout's indices in order, with
    weight_decay, amsgrad and maximize off, and a state for every parameter with one common step, or none at all."""
    groups = sd.get("param_groups", [])
    if len(groups) != 1 or list(groups[0]["params"]) != [i for i, _, _ in layout]:
        raise ValueError("expected one param group over model.parameters() in order")
    g = groups[0]
    if g.get("weight_decay", 0) or g.get("amsgrad", False) or g.get("maximize", False):
        raise ValueError("weight_decay, amsgrad and maximize are not part of the fused Adam")
    betas, eps = _adam_hyper(tuple(g["betas"]), g["eps"])
    state = sd.get("state", {})
    steps = {float(st["step"]) for st in state.values()}
    if state and (set(state) != {i for i, _, _ in layout} or len(steps) != 1):
        raise ValueError("every parameter needs a state, all with one common step")
    step = steps.pop() if state else 0.0
    if step != int(step) or step < 0:
        raise ValueError(f"step must be a whole number >= 0, got {step}")
    for i, shape, _ in layout if state else []:
        for key in ("exp_avg", "exp_avg_sq"):
            if tuple(state[i][key].shape) != shape:
                raise ValueError(f"state {i} {key}: shape {tuple(state[i][key].shape)}, expected {shape}")
    with torch.no_grad():
        if not state:
            flat_m.zero_(); flat_v.zero_()
        for i, shape, off in layout if state else []:
            n = math.prod(shape)
            flat_m[off:off + n].view(shape).copy_(state[i]["exp_avg"])
            flat_v[off:off + n].view(shape).copy_(state[i]["exp_avg_sq"])
    return int(step), betas, eps, float(g.get("lr", 1e-3))


class Trainer:
    def __init__(self, model: Model, batch_size: int, seq_length: int, process_group=None,
                 keep_clipped_grads: bool = False, data_parallel: bool = True, lazy_update: bool = False, *,
                 ar: float = 0.0, tar: float = 0.0, optimizer: str = "sgd", betas=(0.9, 0.999), eps: float = 1e-8):
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
        gradients of the step; weights, loss and norm are the same either way.
        ar / tar (keyword only): AWD-LSTM's activation regularization (Merity et al. 2018; DESIGN.md section 17), alpha
        and beta >= 0.  Every fused train step adds alpha/(T*H) * sum(y^2) over the last layer's dropped output y and
        beta/((T-1)*H) * sum((h_t - h_{t-1})^2) over its raw output h (AWD's main.py terms, times B) to the loss it
        differentiates; the clip norm and `.grad` include their gradient.  The returned loss stays the NLL;
        `activation_reg` holds the two penalty values of the last step.  Eval calls ignore them.
        optimizer / betas / eps (keyword only): "sgd" (default) or "adam" (Kingma & Ba 2015; DESIGN.md section 21), the
        update every train step applies after the global-norm clip, lr being the train step's own.  Adam is
        torch.optim.Adam(betas=betas, eps=eps, weight_decay=0): the moments live in `flat_m` and `flat_v` (flat_p's
        layout), the update count in `adam_step`; `optimizer_state_dict()` / `load_optimizer_state_dict()` move them
        to and from torch.optim.Adam's format.  Iterate averaging is an SGD scheme and refuses to start under Adam."""
        for name, v in (("ar", ar), ("tar", tar)):
            if isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) or v < 0:
                raise ValueError(f"{name} must be a finite number >= 0, got {v!r}")
        self._ar, self._tar = float(ar), float(tar)
        if optimizer not in ("sgd", "adam"):
            raise ValueError(f"optimizer must be 'sgd' or 'adam', got {optimizer!r}")
        self.optimizer = optimizer
        self._betas, self._eps = _adam_hyper(betas, eps)
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
        if model.experts and self.world > 1:
            raise ValueError("a Mixture-of-Softmaxes model does not train data parallel yet: "
                             "create the Trainer with data_parallel=False")
        params = model.ordered_parameters()
        head = params[len(params) - 3:] if model.experts else []   # the Mixture-of-Softmaxes head, laid out last
        base = params[:len(params) - len(head)]
        # flat layout: the library's order, except that a tied E sits next to fc.b, so that the bucket the projection
        # backward completes (E's G_proj part, fc.b) is one range
        layout = (base[1:-1] + [base[0], base[-1]] if model.tied else base) + head
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
        self._reg = torch.zeros(2, device=dev)
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
        self.adam_step = 0             # Adam: the updates applied so far (torch.optim.Adam's state "step")
        if optimizer == "adam":
            self.flat_m = torch.zeros_like(self.flat_p)
            self.flat_v = torch.zeros_like(self.flat_p)
            self._m_s = self._flat_params_struct(self.flat_m)
            self._v_s = self._flat_params_struct(self.flat_v)
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
            E, N = model.embed_size, batch_size * seq_length    # embedding rows are E wide
            self._rows = torch.zeros(N, E, device=dev)
            self._rows_all = torch.zeros(self.world * N, E, device=dev)
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
        requested, and a fresh context must be told that the weights are new to it and get the Trainer's modes).  A
        fresh context holds no average: one found while averaging is on stops the averaging and raises RuntimeError
        (the model refuses to re-create its context while a Trainer averages, so only a context dropped some other
        way gets here)."""
        c = self.model._context(self.T, self.B)
        if self._ctx_cached != self.model._ctx_serial:
            _lib.check(_lib.load().zrb_params_changed(c))
            _lib.check(_lib.load().zrb_set_embed_sparse(c, int(getattr(self, "_embed_sparse", 0))))
            _lib.check(_lib.load().zrb_set_keep_clipped_grads(c, 1 if self._keep_clipped else 0))
            _lib.check(_lib.load().zrb_set_lazy_update(c, 1 if getattr(self, "_lazy", False) else 0))
            _lib.check(_lib.load().zrb_set_activation_reg(c, self._ar, self._tar))
            if getattr(self, "optimizer", "sgd") == "adam":
                self._set_adam(c)
            self._ctx_cached = self.model._ctx_serial
            if getattr(self, "_averaging", False):
                self._set_averaging(False)
                raise RuntimeError("the model's library context was re-created while averaging was on: the average "
                                   "stops here (flat_avg holds it as it was); call start_averaging() to restart")
        return c

    def _set_adam(self, c):
        """Hand Adam's moments, hyper-parameters and update count to the context c."""
        _lib.check(_lib.load().zrb_set_adam(c, C.byref(self._m_s), C.byref(self._v_s), self._betas[0], self._betas[1],
                                            self._eps, self.adam_step))

    def _set_averaging(self, on):
        """Whether averaging is on; while it is, the model keeps its library context (the average's count lives there)."""
        self._averaging = on
        self.model._ctx_pinned = "the Trainer's running average (start_averaging)" if on else None

    @property
    def activation_reg(self):
        """CUDA tensor [2]: the alpha-weighted AR and beta-weighted TAR values of the last train step (zeros while both
        are off), copied on the Trainer's stream without a host synchronisation."""
        _lib.check(_lib.load().zrb_activation_reg(self.ctx, _lib.ptr(self._reg), self._stream()))
        return self._reg

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

    # ---- main.py:109-117 -----------------------------------------------------------------
    def train_step(self, x, y, lr, max_norm):
        """x, y: [T,B] int64 CUDA tensors (contiguous).  Returns (loss, norm) as 0-d CUDA
        tensors (no host sync)."""
        lib = _lib.load()
        T, B = x.shape
        self._check_not_swapped()
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
        self._updated(lr)
        return self.loss, self.norm

    def _updated(self, lr):
        self._pending = True
        self._lr = float(lr)
        if self.optimizer == "adam":
            self.adam_step += 1

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
        self._check_not_swapped()
        if self.world == 1:
            self._check_versions()
            _lib.check(lib.zrb_train_step_host(self.ctx, C.byref(self._ps), C.byref(self._gs),
                                               C.c_void_p(hx.data_ptr()), C.c_void_p(hy.data_ptr()), T, B,
                                               C.byref(self._st), C.byref(self._st), self.seed, self.step,
                                               float(lr), float(max_norm), C.c_void_p(self._hloss.data_ptr()),
                                               C.c_void_p(self._hloss.data_ptr() + 4), self._stream()))
            self.step += 1
            self._updated(lr)
            return float(self._hloss[0]), float(self._hloss[1])
        xd = hx.to(self.dev, non_blocking=True); yd = hy.to(self.dev, non_blocking=True)
        loss, norm = self.train_step(xd, yd, lr, max_norm)
        both = torch.stack([loss, norm]).cpu()
        return float(both[0]), float(both[1])

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
            self._no_experts("the neural cache")
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
        if cache is not None:
            self._no_experts("the neural cache")
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

    # ---- iterate averaging, NT-ASGD (DESIGN.md section 16) -----------------------------------------------------------
    def _check_not_swapped(self):
        if getattr(self, "_swapped", False):
            raise RuntimeError("train_step inside averaged_weights(): the parameters hold the average")

    def start_averaging(self):
        """Average the weights over every following train step (zrb_set_average): after n steps `flat_avg` holds the
        mean of the n weight vectors those steps produced, as torch.optim.ASGD(lambd=0, t0=0) created now would.  The
        weights themselves train exactly as without averaging.  Calling it again restarts at n = 0.  Under data
        parallelism every rank calls it at the same step (the ranks' averages stay identical; nothing is exchanged).
        ValueError under Adam: NT-ASGD averages SGD iterates."""
        if self.optimizer == "adam":
            raise ValueError("iterate averaging (NT-ASGD) is an SGD scheme: it does not run with optimizer='adam'")
        self._check_not_swapped()
        if getattr(self, "flat_avg", None) is None:
            self.flat_avg = torch.zeros_like(self.flat_p)
        self._avg_s = self._flat_params_struct(self.flat_avg)
        self.flush()
        _lib.check(_lib.load().zrb_set_average(self.ctx, C.byref(self._avg_s)))
        self._set_averaging(True)

    def stop_averaging(self):
        """Stop averaging; `flat_avg` keeps the average so far."""
        self._check_not_swapped()
        self.flush()
        _lib.check(_lib.load().zrb_set_average(self.ctx, None))
        self._set_averaging(False)

    @property
    def averaged_steps(self):
        """n: the train steps averaged since start_averaging() (0 while averaging is off)."""
        n = C.c_int64()
        _lib.check(_lib.load().zrb_average_count(self.ctx, C.byref(n)))
        return n.value

    @contextlib.contextmanager
    def averaged_weights(self):
        """`with trainer.averaged_weights():` the parameters hold the average (zrb_swap_average exchanges them with
        `flat_avg` and rebuilds the fp16 weight images in the same pass); perplexity, eval_step, generation, beam search,
        the cache and dynamic evaluation see it.  On exit the weights are swapped back bit for bit.  train_step inside the
        block raises RuntimeError."""
        self._check_not_swapped()
        lib = _lib.load()
        self.flush()
        self._check_versions()
        _lib.check(lib.zrb_swap_average(self.ctx, C.byref(self._ps), self._stream()))
        serial = self.model._ctx_serial
        self._swapped = True
        try:
            yield self
        finally:
            if self.model._ctx is not None and self.model._ctx_serial == serial:
                self.flush()
                self._check_versions()
                _lib.check(lib.zrb_swap_average(self.ctx, C.byref(self._ps), self._stream()))
                self._swapped = False
            else:
                # the context was dropped inside the block and its successor holds no average to swap back: exchange
                # the two buffers with copies, then have the weights repacked (which reports the lost average)
                with torch.no_grad():
                    trained = self.flat_avg.clone()
                    self.flat_avg.copy_(self.flat_p)
                    self.flat_p.copy_(trained)
                self._swapped = False
                self.params_changed()

    def average_state_dict(self):
        """The average as a state dict under the model's own keys (tied: embed.W and fc.W both, as state_dict()
        gives them): what AWD-LSTM saves as its final model.  Copies; pending updates are applied first."""
        if getattr(self, "flat_avg", None) is None or self.averaged_steps == 0:
            raise RuntimeError("no average: call start_averaging() and train at least one step")
        self.flush()
        base, n = self.flat_p.data_ptr(), self.flat_p.numel()
        src = self.flat_p if getattr(self, "_swapped", False) else self.flat_avg
        out = {}
        for k, v in self.model.state_dict().items():
            off = (v.data_ptr() - base) // 4
            if v.dtype == torch.float32 and 0 <= off < n:
                v = src[off:off + v.numel()].view_as(v)
            out[k] = v.detach().clone()
        return out

    # ---- Adam (DESIGN.md section 21) ---------------------------------------------------------------------------------
    def _adam_layout(self):
        """(index, shape, offset into flat_p) in model.parameters() order: torch.optim.Adam's state indices."""
        if self.optimizer != "adam":
            raise ValueError("the Trainer was created with optimizer='sgd': there is no Adam state")
        base = self.flat_p.data_ptr()
        return [(i, tuple(p.shape), (p.data_ptr() - base) // 4) for i, p in enumerate(self.model.parameters())]

    def optimizer_state_dict(self):
        """Adam's state in torch.optim.Adam's state_dict() format for an Adam over model.parameters() (copies on the
        parameters' device), with one param group of the betas, eps and the last train step's lr.  Pending lazy updates
        are applied first."""
        layout = self._adam_layout()
        self.flush()
        return adam_state_to_torch(self.flat_m, self.flat_v, self.adam_step, layout, getattr(self, "_lr", 1e-3),
                                   self._betas, self._eps)

    def load_optimizer_state_dict(self, sd):
        """Load a torch.optim.Adam state_dict() over model.parameters() (or one from optimizer_state_dict()): the
        moments, the update count, and the group's betas, eps and lr (see adam_state_from_torch).  Pending lazy updates
        are applied first."""
        layout = self._adam_layout()
        self.flush()
        self.adam_step, self._betas, self._eps, lr = adam_state_from_torch(sd, layout, self.flat_m, self.flat_v)
        self._lr = lr
        self._set_adam(self.ctx)

    # ---- dynamic evaluation (DESIGN.md section 14) -------------------------------------------------------------------
    def _no_experts(self, what):
        if self.model.experts:
            raise ValueError(f"{what} does not support a Mixture-of-Softmaxes model (experts={self.model.experts}) yet")

    def _single_replica(self, what):
        self._no_experts(what)
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
        depends only on the model).  While averaging is on (or inside averaged_weights()) larger windows raise
        ValueError before anything changes: the average lives in the context.  Returns a `GradStats`."""
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
        T_ctx, B_ctx = self.model._ctx_key[:2]
        if (T > T_ctx or B > B_ctx) and getattr(self, "_averaging", False):
            raise ValueError(f"[T={T}, B={B}] windows need a larger library context than [{T_ctx}, {B_ctx}], and "
                             "re-creating it would lose the running average: compute the statistics on a Trainer of "
                             "their shape")
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
