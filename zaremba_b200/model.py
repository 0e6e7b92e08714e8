"""Drop-in replacement for the reference's `model.py` (`from model import Model`).

Same constructor arguments, parameter names / shapes / registration order, RNG
consumption at construction, `(h, c)` state layouts and `forward(x, states)` contract as
/root/reference/model.py:75-110 -- but every tensor operation of the forward and backward
pass runs in libzaremba_b200.so (hand-written sm_90a CUDA behind the C ABI of
include/zaremba_b200.h).  PyTorch is used for device memory, streams and autograd glue
only.  There is no CPU path: the module refuses to run off a CUDA device.

Reference lines mirrored:
  Embed / LSTM / Linear containers   model.py:6-71   (parameter holders here; names kept)
  Model.__init__ / reset_parameters  model.py:76-92
  state_init / detach                model.py:94-101
  forward                            model.py:103-110
"""
from __future__ import annotations

import ctypes as C
import math
import operator

import torch
from torch import nn

from . import _lib


class Embed(nn.Module):
    """Parameter holder for `embed.W` [V,E] (model.py:6-17; E = H unless `Model(embed_size=E)`)."""

    def __init__(self, vocab_size, embed_size):
        super().__init__()
        self.vocab_size, self.embed_size = vocab_size, embed_size
        self.W = nn.Parameter(torch.empty(vocab_size, embed_size))

    def extra_repr(self):
        return f"vocab: {self.vocab_size}, embedding: {self.embed_size}"


class LSTM(nn.Module):
    """Parameter holder for one recurrent layer.

    lstm_type "pytorch": torch.nn.LSTM names and gate order (i,f,g,o) (model.py:84);
    constructing it consumes the global RNG exactly like nn.LSTM(input_size, hidden_size).__init__
    does (four U(-1/sqrt(H), 1/sqrt(H)) draws: [4H,In], [4H,H], [4H], [4H]), so that a seeded
    `Model(...)` gets the reference's weights.  lstm_type "custom": the reference's own cell
    (model.py:20-31): names W_x/W_h/b_x/b_h, row blocks (i,f,o,n), no RNG consumption, H->H only.
    """

    def __init__(self, input_size, hidden_size, lstm_type="pytorch"):
        super().__init__()
        if lstm_type == "custom" and input_size != hidden_size:
            raise ValueError("lstm_type 'custom' builds H->H layers only")
        self.input_size, self.hidden_size, self.lstm_type = input_size, hidden_size, lstm_type
        H, In = hidden_size, input_size
        if lstm_type == "custom":
            self.W_x = nn.Parameter(torch.empty(4 * H, H))
            self.W_h = nn.Parameter(torch.empty(4 * H, H))
            self.b_x = nn.Parameter(torch.empty(4 * H))
            self.b_h = nn.Parameter(torch.empty(4 * H))
        else:
            stdv = 1.0 / math.sqrt(H)
            self.weight_ih_l0 = nn.Parameter(torch.empty(4 * H, In).uniform_(-stdv, stdv))
            self.weight_hh_l0 = nn.Parameter(torch.empty(4 * H, H).uniform_(-stdv, stdv))
            self.bias_ih_l0 = nn.Parameter(torch.empty(4 * H).uniform_(-stdv, stdv))
            self.bias_hh_l0 = nn.Parameter(torch.empty(4 * H).uniform_(-stdv, stdv))

    def tensors(self):
        if self.lstm_type == "custom":
            return self.W_x, self.W_h, self.b_x, self.b_h
        return self.weight_ih_l0, self.weight_hh_l0, self.bias_ih_l0, self.bias_hh_l0

    def extra_repr(self):
        return f"input: {self.input_size}, hidden: {self.hidden_size}, type: {self.lstm_type}"


class Linear(nn.Module):
    """Parameter holder for `fc.W` [V,H_{L-1}], `fc.b` [V] (model.py:57-71)."""

    def __init__(self, input_size, hidden_size):
        super().__init__()
        self.input_size, self.hidden_size = input_size, hidden_size
        self.W = nn.Parameter(torch.empty(hidden_size, input_size))
        self.b = nn.Parameter(torch.empty(hidden_size))

    def extra_repr(self):
        return f"input: {self.input_size}, output: {self.hidden_size}"


class Prior(nn.Module):
    """Parameter holder for `prior.W` [K,H_{L-1}] of a Mixture-of-Softmaxes head (no bias)."""

    def __init__(self, input_size, experts):
        super().__init__()
        self.input_size, self.experts = input_size, experts
        self.W = nn.Parameter(torch.empty(experts, input_size))

    def extra_repr(self):
        return f"input: {self.input_size}, experts: {self.experts}"


def _check_widths(hidden_size, layer_num, embed_size, layer_sizes):
    """(E, layer widths) of a Model, or ValueError"""
    def width(v, what):
        try:
            n = operator.index(v)
        except TypeError:
            n = 0
        if isinstance(v, bool) or n < 1:
            raise ValueError(f"{what} must be a positive int, got {v!r}")
        return n
    H = width(hidden_size, "hidden_size")
    E = H if embed_size is None else width(embed_size, "embed_size")
    if layer_sizes is None:
        return E, (H,) * layer_num
    sizes = tuple(width(v, "every entry of layer_sizes") for v in layer_sizes)
    if len(sizes) != layer_num:
        raise ValueError(f"layer_sizes has {len(sizes)} entries for {layer_num} layers")
    if sizes[0] != H:
        raise ValueError(f"hidden_size ({H}) must equal layer_sizes[0] ({sizes[0]})")
    return E, sizes


def model_from_state_dict(state_dict, dropout=0.0, winit=0.0, tied=None, **kwargs):
    """A `Model` shaped like `state_dict` (pytorch layout) with its values loaded: V and E from `embed.W`, the layer
    widths from each `rnns.l.weight_hh_l0`, tied (None) when `fc.W` equals `embed.W`.  kwargs go to `Model`."""
    E_w = torch.as_tensor(state_dict["embed.W"])
    V, E = E_w.shape
    sizes, l = [], 0
    while f"rnns.{l}.weight_hh_l0" in state_dict:
        sizes.append(int(torch.as_tensor(state_dict[f"rnns.{l}.weight_hh_l0"]).shape[1]))
        l += 1
    if not sizes:
        raise ValueError("state_dict has no rnns.<l>.weight_hh_l0 (lstm_type 'pytorch' layout expected)")
    fc_w = torch.as_tensor(state_dict["fc.W"])
    if tied is None:
        tied = fc_w.shape == E_w.shape and torch.equal(fc_w.cpu(), E_w.cpu())
    if "prior.W" in state_dict:   # a Mixture-of-Softmaxes head: K from prior.W
        kwargs.setdefault("experts", int(torch.as_tensor(state_dict["prior.W"]).shape[0]))
    m = Model(int(V), sizes[0], len(sizes), dropout, winit, tied=tied, embed_size=int(E), layer_sizes=tuple(sizes),
              **kwargs)
    m.load_state_dict(state_dict)
    return m


def _ifon_to_ifgo(t):
    """custom cell row blocks (i,f,o,n) <-> nn.LSTM (i,f,g,o); the permutation is an involution."""
    i, f, a, b = t.chunk(4, 0)
    return torch.cat([i, f, b, a], 0)


class _LmFunction(torch.autograd.Function):
    """autograd node for model.py:103-110: forward = zrb_forward, backward = zrb_backward."""

    @staticmethod
    def forward(ctx, model, x_dev, states_in, seed, step, *weights):
        scores, states_out = model._run_forward(x_dev, states_in, weights, seed, step, want_scores=True)
        ctx.model = model
        ctx.fwd_id = model._fwd_id
        ctx.save_for_backward(*weights)
        flat = [t for hc in states_out for t in hc]
        ctx.mark_non_differentiable(*flat)
        return (scores, *flat)

    @staticmethod
    def backward(ctx, dscores, *unused):
        model = ctx.model
        if ctx.fwd_id != model._fwd_id:
            raise RuntimeError("zaremba_b200.Model keeps activations of the latest forward only; "
                               "backward() must follow the forward it belongs to")
        grads = model._run_backward(dscores.contiguous(), ctx.saved_tensors)
        return (None, None, None, None, None, *grads)


class Model(nn.Module):
    """`Model(vocab_size, hidden_size, layer_num, dropout, winit, lstm_type="pytorch")`.

    Extra keyword `engine`: "tc" (wgmma tensor cores, default) or "simt" (fp32 CUDA cores,
    validation).

    Extra keywords `variational` / `recurrent_dropout`: variational dropout (Gal & Ghahramani 2016; DESIGN.md
    section 11).  With `variational=True` every dropout mask is drawn once per window and reused at every time step,
    and the recurrent connection of each layer is dropped with p = `recurrent_dropout` (None: the same p as
    `dropout`, Gal's setting; 0: no recurrent dropout).  Eval mode applies no mask either way.

    Extra keyword `tied`: tie the embedding and softmax weights (Press & Wolf 2017; DESIGN.md section 13).  `fc.W` is
    then the same `nn.Parameter` as `embed.W` (one [V,H] matrix E, `fc.b` stays separate), `parameters()` yields the
    2 + 4L distinct tensors, and the library takes E's one merged gradient.  `reset_parameters` walks `parameters()`,
    so with the same seed E and the LSTM tensors equal an untied model's `embed.W` and LSTM tensors, and `fc.b` is
    drawn where the untied model draws `fc.W`.  `state_dict()` carries both keys (torch's rule for a shared parameter),
    so a tied checkpoint also loads into an untied model; loading one whose `embed.W` and `fc.W` differ into a tied
    model raises ValueError.

    Extra keyword `weight_drop`: the weight-dropped LSTM (Merity et al. 2018; DESIGN.md section 15), DropConnect with
    this p on every layer's hidden-to-hidden matrix.  In train mode each forward draws one mask per layer and uses
    W_hh * mask / (1 - p) at every time step; the gradient reaching `weight_hh_l0` is masked alike.  Eval mode uses the
    raw W_hh.  The masks are seeded by `torch.initial_seed()` when the library context is created (no rank in it: every
    data-parallel rank draws the same mask).  Not with lstm_type "custom".

    Extra keyword `embed_dropout`: embedding dropout (Merity et al. 2018; DESIGN.md section 17), whole word types
    dropped with this p.  In train mode each forward draws one keep flag per vocabulary row and gathers the kept rows
    of `embed.W` scaled by 1 / (1 - p), before the dropout after the embedding; the gradient reaching `embed.W` is
    masked alike.  Tied: only the lookup is masked, the projection uses the raw matrix.  Eval mode, `generate` and
    `beam_search` use the raw rows.  Seeded like `weight_drop` (no rank in it).

    Extra keywords `embed_size` / `layer_sizes`: layers of unequal width (DESIGN.md section 18), e.g. AWD-LSTM's PTB
    model `Model(10000, 1150, 3, p, winit, tied=True, embed_size=400, layer_sizes=(1150, 1150, 400))`.  `embed.W` is
    [V,E], layer l is an nn.LSTM(In_l, H_l) with In_0 = E and In_l = H_{l-1}, `fc.W` is [V,H_{L-1}], and the states of
    layer l are [1,B,H_l].  `embed_size` defaults to `hidden_size`, `layer_sizes` to (hidden_size,) * layer_num; given,
    it has layer_num entries and the first is `hidden_size`.  `tied=True` needs E = H_{L-1}.  Unequal widths take the
    tensor-core engine and lstm_type "pytorch".  With every width equal this is the model above, bit for bit.

    Extra keywords `experts` / `mos_dropout`: a Mixture-of-Softmaxes head (Yang et al. 2018; DESIGN.md section 19),
    e.g. the PTB model `Model(10000, 960, 3, p, winit, tied=True, embed_size=280, layer_sizes=(960, 960, 620),
    experts=15)`.  With h the last layer's output after its dropout, `latent.W` [K*E,H_{L-1}] and `latent.b` [K*E] give K
    latent vectors c_k = tanh(latent(h))_k (dropped with p = `mos_dropout` in train mode), `prior.W` [K,H_{L-1}] (no bias)
    the mixture weights pi = softmax(h prior.W^T), and `fc` [V,E] each expert's softmax; forward returns
    log(sum_k pi_k softmax(fc(c_k))) [T*B,V], so nn.CrossEntropyLoss on it is the exact NLL, and `generate` /
    `beam_search` sample from the mixture.  The three head tensors are registered after `fc`, so with the same seed the
    other tensors equal the plain model's.  `tied=True` needs nothing beyond E.  Not with engine "simt", lstm_type
    "custom", data parallel, the neural cache or dynamic evaluation (ValueError).

    Extra keywords `zoneout_cell` / `zoneout_hidden`: zoneout (Krueger et al. 2017; DESIGN.md section 20).  In train
    mode each unit of every layer keeps its previous c with probability `zoneout_cell` and its previous h with
    probability `zoneout_hidden` at each time step, instead of taking the new values; eval mode (and `generate`,
    `beam_search`) uses the expectation z * previous + (1 - z) * new.  The flags are seeded like dropout.  Not with
    lstm_type "custom" or engine "simt" (ValueError).  `state_dict()` is unchanged.
    """

    def __init__(self, vocab_size, hidden_size, layer_num, dropout, winit, lstm_type="pytorch", engine="tc",
                 variational=False, recurrent_dropout=None, *, tied=False, weight_drop=0.0, embed_dropout=0.0,
                 embed_size=None, layer_sizes=None, experts=None, mos_dropout=0.0, zoneout_cell=0.0,
                 zoneout_hidden=0.0):
        super().__init__()
        E, sizes = _check_widths(hidden_size, layer_num, embed_size, layer_sizes)
        equal = all(w == E for w in sizes)
        if experts is not None:
            if isinstance(experts, bool) or not isinstance(experts, int) or not 1 <= experts <= _lib.MAX_EXPERTS:
                raise ValueError(f"experts must be an int in [1, {_lib.MAX_EXPERTS}], got {experts!r}")
            if engine == "simt":
                raise ValueError("a Mixture-of-Softmaxes head needs the tensor-core engine (engine='tc')")
            if lstm_type == "custom":
                raise ValueError("a Mixture-of-Softmaxes head needs lstm_type 'pytorch'")
            if layer_num > 3:
                raise ValueError("a Mixture-of-Softmaxes model takes at most 3 layers")
        if isinstance(mos_dropout, bool) or not isinstance(mos_dropout, (int, float)) or \
                not 0.0 <= float(mos_dropout) < 1.0:
            raise ValueError(f"mos_dropout must be a number in [0, 1), got {mos_dropout!r}")
        if mos_dropout and experts is None:
            raise ValueError("mos_dropout needs experts")
        for name, z in (("zoneout_cell", zoneout_cell), ("zoneout_hidden", zoneout_hidden)):
            if isinstance(z, bool) or not isinstance(z, (int, float)) or not 0.0 <= float(z) < 1.0:
                raise ValueError(f"{name} must be a number in [0, 1), got {z!r}")
        if zoneout_cell or zoneout_hidden:
            if lstm_type == "custom":
                raise ValueError("zoneout needs lstm_type 'pytorch'")
            if engine == "simt":
                raise ValueError("zoneout needs the tensor-core engine (engine='tc')")
        if not equal and lstm_type == "custom":
            raise ValueError("layers of unequal width need lstm_type 'pytorch'")
        if not equal and engine == "simt":
            raise ValueError("layers of unequal width need the tensor-core engine (engine='tc')")
        if tied and E != sizes[-1] and experts is None:
            raise ValueError(f"tied=True needs embed_size = layer_sizes[-1] (got {E} and {sizes[-1]})")
        if lstm_type not in ("pytorch", "custom"):
            raise ValueError(f"lstm_type must be 'pytorch' or 'custom', got {lstm_type!r}")
        if isinstance(weight_drop, bool) or not isinstance(weight_drop, (int, float)) or \
                not 0.0 <= float(weight_drop) < 1.0:
            raise ValueError(f"weight_drop must be a number in [0, 1), got {weight_drop!r}")
        if isinstance(embed_dropout, bool) or not isinstance(embed_dropout, (int, float)) or \
                not 0.0 <= float(embed_dropout) < 1.0:
            raise ValueError(f"embed_dropout must be a number in [0, 1), got {embed_dropout!r}")
        if weight_drop and lstm_type == "custom":
            raise ValueError("weight_drop applies to lstm_type 'pytorch' only")
        if variational not in (False, True):
            raise ValueError(f"variational must be True or False, got {variational!r}")
        if not isinstance(tied, bool):
            raise ValueError(f"tied must be True or False, got {tied!r}")
        if recurrent_dropout is not None and not variational:
            raise ValueError("recurrent_dropout needs variational=True")
        p_rec = float(dropout) if (variational and recurrent_dropout is None) else float(recurrent_dropout or 0.0)
        if not 0.0 <= p_rec < 1.0:
            raise ValueError(f"recurrent_dropout must be in [0, 1), got {recurrent_dropout!r}")
        if layer_num > _lib.MAX_LAYERS:
            raise ValueError(f"at most {_lib.MAX_LAYERS} layers")
        self.vocab_size = vocab_size
        self.hidden_size = hidden_size
        self.layer_num = layer_num
        self.winit = winit
        self.lstm_type = lstm_type
        self.engine = engine
        self.p_drop = float(dropout)
        self.variational = bool(variational)
        self.p_rec = p_rec
        self.tied = tied
        self.weight_drop = float(weight_drop)
        self.embed_dropout = float(embed_dropout)
        self.embed_size = E
        self.layer_sizes = sizes
        self._widths_given = embed_size is not None or layer_sizes is not None
        self.experts = experts
        self.mos_dropout = float(mos_dropout)
        self.zoneout_cell = float(zoneout_cell)
        self.zoneout_hidden = float(zoneout_hidden)
        self.embed = Embed(vocab_size, E)
        self.rnns = nn.ModuleList(LSTM(([E] + list(sizes))[l], sizes[l], lstm_type) for l in range(layer_num))
        self.fc = Linear(E if experts else sizes[-1], vocab_size)
        if tied:
            self.fc.W = self.embed.W
        if experts:   # after fc: a seeded model's other tensors equal the plain model's
            self.prior = Prior(sizes[-1], experts)
            self.latent = Linear(sizes[-1], experts * E)
        self.dropout = nn.Dropout(p=dropout)     # kept for repr / state parity; masks come from the library
        self.reset_parameters()
        self._ctx = None
        self._ctx_key = None
        self._ctx_serial = 0           # contexts created so far
        self._ctx_pinned = None        # what a re-created context would lose (a Trainer's average), or None
        self._fwd_id = 0
        self._drop_step = 0
        self._seed = None
        self._versions = None
        self._explicit_masks = None

    # ---- reference API -----------------------------------------------------------------
    def reset_parameters(self):
        for param in self.parameters():          # model.py:90-92
            nn.init.uniform_(param, -self.winit, self.winit)

    def state_init(self, batch_size):
        dev = next(self.parameters()).device
        return [(torch.zeros(s, device=dev), torch.zeros(s, device=dev)) for s in self._state_shapes(batch_size)]

    def _state_shapes(self, batch_size):
        """the (h, c) shape of every layer for `batch_size` rows"""
        if self.lstm_type == "custom":
            return [(batch_size, H) for H in self.layer_sizes]
        return [(1, batch_size, H) for H in self.layer_sizes]

    def detach(self, states):
        return [(h.detach(), c.detach()) for (h, c) in states]

    def load_state_dict(self, state_dict, strict=True, assign=False):
        if self.tied and "embed.W" in state_dict and "fc.W" in state_dict and \
                not torch.equal(torch.as_tensor(state_dict["embed.W"]).cpu(), torch.as_tensor(state_dict["fc.W"]).cpu()):
            raise ValueError("checkpoint has different embed.W and fc.W: it cannot load into a tied model (tied=True)")
        return super().load_state_dict(state_dict, strict=strict, assign=assign)

    def forward(self, x, states):
        dev = self.embed.W.device
        if dev.type != "cuda":
            raise RuntimeError("zaremba_b200.Model runs on a CUDA device only (no CPU fallback): call .to('cuda')")
        x_dev = x.to(device=dev, dtype=torch.int64).contiguous()   # main.py hands CPU non-contiguous views
        self._context(*x_dev.shape)    # a window the model cannot take raises before it consumes a dropout step
        weights = self._lib_weights()
        seed, step = self._next_dropout_key()
        need_grad = torch.is_grad_enabled() and any(w.requires_grad for w in weights)
        if need_grad:
            outs = _LmFunction.apply(self, x_dev, states, seed, step, *weights)
            scores, flat = outs[0], outs[1:]
            new_states = [(flat[2 * i], flat[2 * i + 1]) for i in range(self.layer_num)]
        else:
            scores, new_states = self._run_forward(x_dev, states, weights, seed, step, want_scores=True)
        for i in range(self.layer_num):          # the reference mutates the caller's list (model.py:107)
            states[i] = new_states[i]
        return scores, states

    # ---- text generation (zrb_generate) ---------------------------------------------------
    def generate(self, prompt, n_new, states=None, temperature=1.0, top_k=0, top_p=1.0, seed=None, pos=0):
        """Continue the B columns of `prompt` ([T0,B] int64, CPU or CUDA) by `n_new` sampled tokens on the device.

        Prefill and decode loop run in one library call without host synchronisation.  Always eval mode (no dropout,
        whatever `.training` says), no autograd, and the dropout step is not advanced.  `states` (model layout, None =
        zeros) enter before the prompt.  Sampling: see `zaremba_b200.sample`; the uniforms of step k are those of
        position `pos + k`, and `seed=None` draws a seed from torch's global generator.

        Returns (tokens [n_new,B] int64, logprobs [n_new,B] fp32, states).  The returned states are those BEFORE the
        last token is consumed, so `generate(tokens[-1:], m, states, ..., seed=seed, pos=pos + n_new)` continues the
        same stream.  The model's library context is reused, never replaced (a Trainer's context keeps the recurrence
        plans of its own batch): a B above its max_batch raises; a model without one gets a context for (min(T0, 64), B).
        """
        dev = self.embed.W.device
        if dev.type != "cuda":
            raise RuntimeError("zaremba_b200.Model runs on a CUDA device only (no CPU fallback): call .to('cuda')")
        x = torch.as_tensor(prompt).to(device=dev, dtype=torch.int64).contiguous()
        if x.dim() != 2 or x.numel() == 0:
            raise ValueError(f"prompt must be a non-empty [T0,B] tensor, got shape {tuple(x.shape)}")
        if int(n_new) < 1:
            raise ValueError(f"n_new must be >= 1, got {n_new}")
        T0, B = x.shape
        if self._ctx is None:
            ctx = self._context(min(T0, 64), B)
        else:
            ctx = self._ctx
            if self._ctx_key[2] != dev.index:
                raise RuntimeError("the model's library context belongs to another device")
            if B > self._ctx_key[1]:
                raise ValueError(f"generate: B={B} exceeds the model's library context (max_batch {self._ctx_key[1]}); "
                                 "generate in batches of at most that many rows")
        if seed is None:
            seed = int(torch.randint(0, 2 ** 63 - 1, (1,)).item())
        from .sampling import sampling_config
        cfg = sampling_config(temperature, top_k, top_p, seed)
        if states is None:
            states = self.state_init(B)
        lib = _lib.load()
        with torch.no_grad():
            self._note_param_versions()
            ps, keep_w = self._params_struct(self._lib_weights())   # custom layout: permuted once per call
            st_in, keep_in = self._states_struct(states)
            out_states = [(torch.empty(s, device=dev), torch.empty(s, device=dev)) for s in self._state_shapes(B)]
            st_out, keep_out = self._states_struct(out_states)
            tokens = torch.empty(int(n_new), B, dtype=torch.int64, device=dev)
            logprobs = torch.empty(int(n_new), B, dtype=torch.float32, device=dev)
            with torch.cuda.device(dev):
                _lib.check(lib.zrb_generate(ctx, C.byref(ps), _lib.ptr(x), T0, B, C.byref(st_in), C.byref(st_out),
                                            int(n_new), C.byref(cfg), int(pos) & 0xFFFFFFFFFFFFFFFF, _lib.ptr(tokens),
                                            _lib.ptr(logprobs), torch.cuda.current_stream(dev).cuda_stream))
        return tokens, logprobs, out_states

    def beam_search(self, prompt, n_new, beams, states=None, eos=None):
        """The `beams` most likely continuations of each column of `prompt` ([T0,B] int64) by `n_new` tokens, ranked
        by the float32 sum of their log-probabilities (zrb_beam_search; DESIGN.md section 10).

        A hypothesis that emits `eos` is finished: it keeps its score, continues with eos at log-probability 0 and
        stays in the ranking.  Raw sums favour short finished hypotheses; re-rank with the returned logprobs for a
        length penalty.  Same rules as `generate`: eval mode, no autograd, the dropout step is not advanced, the context
        is reused and never replaced (B * beams above its max_batch raises); a model without one gets a context for
        (min(T0, 64), B * beams).  `states` (model layout, batch B, None = zeros) enter before the prompt.

        Returns (tokens [n_new,B,K] int64, logprobs [n_new,B,K] fp32, scores [B,K] fp32, states): hypothesis k of
        prompt b, best first; states have batch B*K, row b*K + k, and hold each hypothesis BEFORE its last token.
        """
        dev = self.embed.W.device
        if dev.type != "cuda":
            raise RuntimeError("zaremba_b200.Model runs on a CUDA device only (no CPU fallback): call .to('cuda')")
        x = torch.as_tensor(prompt).to(device=dev, dtype=torch.int64).contiguous()
        if x.dim() != 2 or x.numel() == 0:
            raise ValueError(f"prompt must be a non-empty [T0,B] tensor, got shape {tuple(x.shape)}")
        if int(n_new) < 1:
            raise ValueError(f"n_new must be >= 1, got {n_new}")
        K = int(beams)
        if not 1 <= K <= min(_lib.MAX_BEAMS, self.vocab_size):
            raise ValueError(f"beams must be in [1, {min(_lib.MAX_BEAMS, self.vocab_size)}], got {beams}")
        T0, B = x.shape
        if self._ctx is None:
            ctx = self._context(min(T0, 64), B * K)
        else:
            ctx = self._ctx
            if self._ctx_key[2] != dev.index:
                raise RuntimeError("the model's library context belongs to another device")
            if B * K > self._ctx_key[1]:
                raise ValueError(f"beam_search: B*beams={B * K} exceeds the model's library context (max_batch "
                                 f"{self._ctx_key[1]}); search fewer prompts at a time")
        if states is None:
            states = self.state_init(B)
        lib = _lib.load()
        with torch.no_grad():
            self._note_param_versions()
            ps, keep_w = self._params_struct(self._lib_weights())   # custom layout: permuted once per call
            st_in, keep_in = self._states_struct(states)
            out_states = [(torch.empty(s, device=dev), torch.empty(s, device=dev)) for s in self._state_shapes(B * K)]
            st_out, keep_out = self._states_struct(out_states)
            tokens = torch.empty(int(n_new), B, K, dtype=torch.int64, device=dev)
            logprobs = torch.empty(int(n_new), B, K, dtype=torch.float32, device=dev)
            scores = torch.empty(B, K, dtype=torch.float32, device=dev)
            with torch.cuda.device(dev):
                _lib.check(lib.zrb_beam_search(ctx, C.byref(ps), _lib.ptr(x), T0, B, C.byref(st_in), C.byref(st_out),
                                               int(n_new), K, -1 if eos is None else int(eos), _lib.ptr(tokens),
                                               _lib.ptr(logprobs), _lib.ptr(scores),
                                               torch.cuda.current_stream(dev).cuda_stream))
        return tokens, logprobs, scores, out_states

    # ---- plumbing ------------------------------------------------------------------------
    def ordered_parameters(self):
        """The 3+4L tensors in registration order, as the library's zrb_params expects them
        (pytorch names / gate order; the custom layout is permuted by `_lib_weights`).  Tied: the 2+4L distinct
        tensors, E once (no fc.W entry).  With experts, prior.W, latent.W and latent.b follow (zrb_mos_params)."""
        out = [self.embed.W]
        for r in self.rnns:
            out += list(r.tensors())
        out += [self.fc.b] if self.tied else [self.fc.W, self.fc.b]
        if self.experts:
            out += [self.prior.W, self.latent.W, self.latent.b]
        return out

    def _lib_weights(self):
        ws = self.ordered_parameters()
        if self.lstm_type == "custom":
            # (i,f,o,n) -> (i,f,g,o) row-block permutation: a differentiable copy, so autograd
            # routes the gradients back into the custom layout
            ws = [_ifon_to_ifgo(w) if 1 <= i <= 4 * self.layer_num else w for i, w in enumerate(ws)]
        return ws

    def _next_dropout_key(self):
        if self._seed is None:
            self._seed = int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF
        step = self._drop_step
        if self.training:
            self._drop_step += 1
        return self._seed, step

    def set_explicit_dropout_masks(self, masks):
        """Replay given keep-masks (list of L+1 uint8/bool CUDA tensors [T,B,W], W = the site's width) instead of
        Philox; None restores Philox.  Used by parity tests with the reference's masks.  They are Zaremba's per-step
        masks: a model in the variational mode refuses them."""
        if masks is not None and self.variational:
            raise ValueError("explicit dropout masks replay Zaremba's per-step masks; this model uses variational dropout")
        self._explicit_masks = None if masks is None else [m.to(torch.uint8).contiguous() for m in masks]
        if self._ctx is not None:
            self._push_masks()

    def _push_masks(self):
        lib = _lib.load()
        if self._explicit_masks is None:
            _lib.check(lib.zrb_set_explicit_masks(self._ctx, None))
        else:
            arr = (C.c_void_p * (self.layer_num + 1))(*[m.data_ptr() for m in self._explicit_masks])
            _lib.check(lib.zrb_set_explicit_masks(self._ctx, arr))

    def _context(self, T, B):
        key = (max(T, 1), max(B, 1), self.embed.W.device.index)
        if self._ctx is not None:
            ok = self._ctx_key[2] == key[2] and self._ctx_key[0] >= T and self._ctx_key[1] >= B
            if ok:
                return self._ctx
            if self._ctx_pinned:
                raise RuntimeError(f"a [T={T}, B={B}] window needs a larger library context than the model's "
                                   f"[{self._ctx_key[0]}, {self._ctx_key[1]}], and re-creating it would lose "
                                   f"{self._ctx_pinned}")
            # the context holds a lazy Trainer's deferred weight updates: apply them before it goes
            dev = self._ctx_key[2]
            with torch.cuda.device(dev):
                _lib.check(_lib.load().zrb_flush_updates(self._ctx, torch.cuda.current_stream(dev).cuda_stream))
            self._destroy_ctx()
        lib = _lib.load()
        # a model given its widths takes zrb_ctx_create_widths, which equals zrb_ctx_create at equal widths
        widths = [self.embed_size, *self.layer_sizes]
        equal = not self._widths_given
        cfg = _lib.ZrbConfig(self.vocab_size, self.hidden_size if equal else 0, self.layer_num, key[0], key[1],
                             _lib.ENGINE_TC if self.engine == "tc" else _lib.ENGINE_SIMT, self.p_drop,
                             _lib.TIED_EMBEDDING if self.tied else 0)
        h = C.c_void_p()
        with torch.cuda.device(self.embed.W.device):
            if self.experts:
                ws = None if equal else (C.c_int32 * len(widths))(*widths)
                _lib.check(lib.zrb_ctx_create_mos(C.byref(cfg), ws, self.experts, C.byref(h)))
            elif equal:
                _lib.check(lib.zrb_ctx_create(C.byref(cfg), C.byref(h)))
            else:
                _lib.check(lib.zrb_ctx_create_widths(C.byref(cfg), (C.c_int32 * len(widths))(*widths), C.byref(h)))
        self._ctx, self._ctx_key = h, key
        self._ctx_serial += 1          # a new context may reuse the old one's address: this tells them apart
        self._versions = None
        if self.variational:
            _lib.check(lib.zrb_set_variational_dropout(h, 1, self.p_rec))
        if self.weight_drop:
            _lib.check(lib.zrb_set_weight_drop(h, self.weight_drop, int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF))
        if self.embed_dropout:
            _lib.check(lib.zrb_set_embed_dropout(h, self.embed_dropout, int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF))
        if self.mos_dropout:
            _lib.check(lib.zrb_set_mos_dropout(h, self.mos_dropout))
        if self.zoneout_cell or self.zoneout_hidden:
            _lib.check(lib.zrb_set_zoneout(h, self.zoneout_cell, self.zoneout_hidden))
        if self._explicit_masks is not None:
            self._push_masks()
        return self._ctx

    def _destroy_ctx(self):
        if getattr(self, "_ctx", None) is not None:
            _lib.load().zrb_ctx_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self._destroy_ctx()
        except Exception:
            pass

    def _params_struct(self, tensors):
        L = self.layer_num
        ps = _lib.ZrbMosParams() if self.experts else _lib.ZrbParams()
        for t in tensors:
            if t.dtype != torch.float32 or not t.is_cuda:
                raise RuntimeError("parameters must be fp32 CUDA tensors")
        ts = [t if t.is_contiguous() else t.contiguous() for t in tensors]
        ps.embed_w = ts[0].data_ptr()
        for l in range(L):
            ps.w_ih[l] = ts[1 + 4 * l].data_ptr()
            ps.w_hh[l] = ts[2 + 4 * l].data_ptr()
            ps.b_ih[l] = ts[3 + 4 * l].data_ptr()
            ps.b_hh[l] = ts[4 + 4 * l].data_ptr()
        ps.fc_w = ts[0].data_ptr() if self.tied else ts[1 + 4 * L].data_ptr()   # tied: E is fc.W too
        if self.experts:
            ps.prior_w, ps.latent_w, ps.latent_b = (t.data_ptr() for t in ts[-3:])
            ps.fc_b = ts[-4].data_ptr()
        else:
            ps.fc_b = ts[-1].data_ptr()
        return ps, ts

    def _states_struct(self, states):
        st = _lib.ZrbStates()
        keep = []
        for l, (h, c) in enumerate(states):
            h = h.detach().to(torch.float32).contiguous()
            c = c.detach().to(torch.float32).contiguous()
            keep += [h, c]
            st.h[l] = h.data_ptr()
            st.c[l] = c.data_ptr()
        return st, keep

    def _note_param_versions(self):
        """main.py:116-117 updates parameters in place outside the library: tell the context so
        it rebuilds its low-precision weight images."""
        v = tuple((p.data_ptr(), p._version) for p in self.parameters())
        if v != self._versions:
            _lib.check(_lib.load().zrb_params_changed(self._ctx))
            self._versions = v

    def _run_forward(self, x_dev, states, weights, seed, step, want_scores=True):
        lib = _lib.load()
        T, B = x_dev.shape
        ctx = self._context(T, B)
        self._note_param_versions()
        dev = x_dev.device
        ps, keep_w = self._params_struct([w.detach() for w in weights])
        st_in, keep_in = self._states_struct(states)
        out_states = [(torch.empty_like(h, dtype=torch.float32), torch.empty_like(c, dtype=torch.float32))
                      for (h, c) in states]
        st_out, keep_out = self._states_struct(out_states)
        scores = torch.empty(T * B, self.vocab_size, device=dev, dtype=torch.float32) if want_scores else None
        stream = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):
            _lib.check(lib.zrb_forward(ctx, C.byref(ps), _lib.ptr(x_dev), T, B, C.byref(st_in), C.byref(st_out),
                                       _lib.ptr(scores), 1 if self.training else 0, seed, step, stream))
        # _states_struct made contiguous detached aliases of out_states' storage
        self._fwd_id += 1
        return scores, out_states

    def _run_backward(self, dscores, weights):
        lib = _lib.load()
        dev = dscores.device
        ps, keep_w = self._params_struct([w.detach() for w in weights])
        grads = [torch.empty_like(w) for w in weights]
        gs, keep_g = self._params_struct(grads)
        stream = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):
            _lib.check(lib.zrb_backward(self._ctx, C.byref(ps), _lib.ptr(dscores.to(torch.float32)), C.byref(gs),
                                        stream))
        return grads
