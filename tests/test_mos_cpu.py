"""Mixture of Softmaxes without a GPU: the fp64 restatement (tests/_model_oracle.py) against torch autograd of a literal
transcription of Yang et al.'s head on a stack of nn.LSTM, the drop-in backward's formulas against autograd, Model's
parameters, initialisation, checkpoints and argument checks, and the C declarations of the new entry points."""
import ctypes as C
import os
import re

import pytest
import torch
from torch import nn

import zaremba_b200
from zaremba_b200 import _lib
from tests import _model_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MOS_PTB = dict(tied=True, embed_size=280, layer_sizes=(960, 960, 620), experts=15)


class _YangHead(nn.Module):
    """The head of Yang et al.'s model.py: latent = Sequential(Linear(nhidlast, ninp * K), Tanh()), prior =
    Linear(nhidlast, K, bias=False), decoder = Linear(ninp, V); prob = sum_k softmax(prior) * softmax(decoder(latent)),
    the loss is -log(prob[y])."""

    def __init__(self, H, E, V, K):
        super().__init__()
        self.K, self.E = K, E
        self.latent = nn.Sequential(nn.Linear(H, K * E), nn.Tanh())
        self.prior = nn.Linear(H, K, bias=False)
        self.decoder = nn.Linear(E, V)

    def forward(self, h):
        latent = self.latent(h)
        logit = self.decoder(latent.view(-1, self.E))
        prior = nn.functional.softmax(self.prior(h), -1)
        prob = nn.functional.softmax(logit, -1).view(-1, self.K, logit.shape[-1])
        return torch.log((prob * prior.unsqueeze(2)).sum(1))


def test_oracle_matches_autograd_of_yangs_head_on_nn_lstm():
    torch.manual_seed(5)
    V, E, sizes, K, T, B = 41, 12, (20, 16), 3, 5, 4
    emb = nn.Embedding(V, E).double()
    lstms = nn.ModuleList(nn.LSTM(([E] + list(sizes))[l], sizes[l]) for l in range(2)).double()
    head = _YangHead(sizes[-1], E, V, K).double()
    for p in list(emb.parameters()) + list(lstms.parameters()) + list(head.parameters()):
        nn.init.uniform_(p, -0.3, 0.3)
    x = torch.randint(0, V, (T, B))
    y = torch.randint(0, V, (T, B))
    inp = emb(x)
    for m in lstms:
        inp, _ = m(inp)
    logp_ref = head(inp.reshape(T * B, -1))
    loss_ref = nn.functional.nll_loss(logp_ref, y.reshape(-1)) * B
    loss_ref.backward()

    params = {"embed.W": emb.weight.detach()}
    for l, m in enumerate(lstms):
        for n in ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0"):
            params[f"rnns.{l}.{n}"] = getattr(m, n).detach()
    params.update({"fc.W": head.decoder.weight.detach(), "fc.b": head.decoder.bias.detach(),
                   "prior.W": head.prior.weight.detach(), "latent.W": head.latent[0].weight.detach(),
                   "latent.b": head.latent[0].bias.detach()})
    states = [(torch.zeros(B, H, dtype=torch.float64), torch.zeros(B, H, dtype=torch.float64)) for H in sizes]
    loss, norm, grads, _, _, _ = O.train_step(params, x, y, states, 2, False, 1.0, 1e9)
    assert abs(loss - loss_ref.item()) < 1e-10
    want = {"embed.W": emb.weight.grad, "fc.W": head.decoder.weight.grad, "fc.b": head.decoder.bias.grad,
            "prior.W": head.prior.weight.grad, "latent.W": head.latent[0].weight.grad,
            "latent.b": head.latent[0].bias.grad}
    for l, m in enumerate(lstms):
        for n in ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0"):
            want[f"rnns.{l}.{n}"] = getattr(m, n).grad
    for k, g in want.items():
        assert torch.allclose(grads[k], g, rtol=1e-9, atol=1e-12), k


def test_one_expert_is_the_plain_softmax_of_tanh_latent():
    torch.manual_seed(1)
    N, H, E, V = 6, 8, 5, 13
    h = torch.randn(N, H, dtype=torch.float64)
    ps = {"latent.W": torch.randn(E, H, dtype=torch.float64), "latent.b": torch.randn(E, dtype=torch.float64),
          "prior.W": torch.randn(1, H, dtype=torch.float64), "fc.W": torch.randn(V, E, dtype=torch.float64),
          "fc.b": torch.randn(V, dtype=torch.float64)}
    want = torch.log_softmax(torch.tanh(h @ ps["latent.W"].t() + ps["latent.b"]) @ ps["fc.W"].t() + ps["fc.b"], -1)
    assert torch.allclose(O.head_logp(h, ps, False, 1), want, atol=1e-12)


@pytest.mark.parametrize("K", [1, 4])
def test_dropin_vjp_formulas_match_autograd(K):
    torch.manual_seed(K)
    N, V = 7, 19
    z = torch.randn(N, K, V, dtype=torch.float64, requires_grad=True)
    a = torch.randn(N, K, dtype=torch.float64, requires_grad=True)
    log_pi = torch.log_softmax(a, -1)
    logp = torch.logsumexp(log_pi[:, :, None] + torch.log_softmax(z, -1), dim=1)
    G = torch.randn(N, V, dtype=torch.float64)
    (logp * G).sum().backward()
    dz, da = O.vjp(logp.detach(), z.detach(), log_pi.detach(), G)
    assert torch.allclose(dz, z.grad, atol=1e-12)
    assert torch.allclose(da, a.grad, atol=1e-12)


def test_mos_ptb_parameter_names_shapes_and_order():
    m = zaremba_b200.Model(10000, 960, 3, 0.4, 0.1, **MOS_PTB)
    got = [(k, tuple(v.shape)) for k, v in m.named_parameters()]
    want = [("embed.W", (10000, 280))]
    for l, (In, H) in enumerate([(280, 960), (960, 960), (960, 620)]):
        want += [(f"rnns.{l}.weight_ih_l0", (4 * H, In)), (f"rnns.{l}.weight_hh_l0", (4 * H, H)),
                 (f"rnns.{l}.bias_ih_l0", (4 * H,)), (f"rnns.{l}.bias_hh_l0", (4 * H,))]
    want += [("fc.b", (10000,)), ("prior.W", (15, 620)), ("latent.W", (15 * 280, 620)), ("latent.b", (15 * 280,))]
    assert got == want
    assert m.fc.W is m.embed.W and m.experts == 15
    assert [p.shape for p in m.ordered_parameters()[-4:]] == [(10000,), (15, 620), (4200, 620), (4200,)]
    m2 = zaremba_b200.Model(50, 30, 2, 0.0, 0.1, experts=2)
    assert tuple(m2.fc.W.shape) == (50, 30) and tuple(m2.latent.W.shape) == (60, 30)


@pytest.mark.parametrize("tied", [False, True])
def test_shared_tensors_equal_the_plain_model_seed_for_seed(tied):
    V, E, sizes, winit = 97, 24, (40, 24), 0.08
    torch.manual_seed(11)
    plain = zaremba_b200.Model(V, sizes[0], 2, 0.0, winit, tied=tied, embed_size=E, layer_sizes=sizes)
    torch.manual_seed(11)
    mos = zaremba_b200.Model(V, sizes[0], 2, 0.0, winit, tied=tied, embed_size=E, layer_sizes=sizes, experts=3)
    pp = dict(plain.named_parameters())
    for k, v in mos.named_parameters():
        if k in pp:
            assert torch.equal(v, pp[k]), k
    for k in ("prior.W", "latent.W", "latent.b"):
        w = dict(mos.named_parameters())[k]
        assert w.abs().max() <= winit and w.abs().max() > 0


def test_state_dict_round_trip():
    torch.manual_seed(2)
    m = zaremba_b200.Model(61, 32, 2, 0.0, 0.1, embed_size=16, layer_sizes=(32, 24), experts=4, tied=True)
    m2 = zaremba_b200.model_from_state_dict(m.state_dict())
    assert m2.experts == 4 and m2.tied and m2.embed_size == 16 and m2.layer_sizes == (32, 24)
    for (k, a), (k2, b) in zip(m.state_dict().items(), m2.state_dict().items()):
        assert k == k2 and torch.equal(a, b)


@pytest.mark.parametrize("kwargs, match", [
    (dict(experts=0), "experts"),
    (dict(experts=33), "experts"),
    (dict(experts=2.0), "experts"),
    (dict(experts=True), "experts"),
    (dict(experts=2, engine="simt"), "tensor-core"),
    (dict(experts=2, lstm_type="custom"), "pytorch"),
    (dict(experts=2, mos_dropout=1.0), "mos_dropout"),
    (dict(mos_dropout=0.1), "needs experts"),
])
def test_model_refuses(kwargs, match):
    with pytest.raises(ValueError, match=match):
        zaremba_b200.Model(20, 8, 2, 0.0, 0.1, **kwargs)


def test_four_layers_refused():
    with pytest.raises(ValueError, match="at most 3 layers"):
        zaremba_b200.Model(20, 8, 4, 0.0, 0.1, experts=2)


def test_tied_mos_needs_nothing_beyond_E():
    m = zaremba_b200.Model(20, 8, 2, 0.0, 0.1, tied=True, embed_size=6, layer_sizes=(8, 10), experts=2)
    assert tuple(m.fc.W.shape) == (20, 6) and tuple(m.latent.W.shape) == (12, 10)
    with pytest.raises(ValueError):
        zaremba_b200.Model(20, 8, 2, 0.0, 0.1, tied=True, embed_size=6, layer_sizes=(8, 10))


def test_params_struct_offsets_match_the_header():
    header = open(os.path.join(ROOT, "include", "zaremba_b200.h")).read()
    body = re.search(r"typedef struct \{\s*zrb_params base;(.*?)\} zrb_mos_params;", header, re.S).group(1)
    fields = re.findall(r"float\*\s+(\w+);", body)
    assert fields == ["prior_w", "latent_w", "latent_b"]
    assert _lib.ZrbMosParams.prior_w.offset == C.sizeof(_lib.ZrbParams)
    for i, f in enumerate(fields):
        assert getattr(_lib.ZrbMosParams, f).offset == C.sizeof(_lib.ZrbParams) + 8 * i
    assert C.sizeof(_lib.ZrbMosParams) == C.sizeof(_lib.ZrbParams) + 24
    assert issubclass(_lib.ZrbMosParams, _lib.ZrbParams)
    assert int(re.search(r"#define ZRB_MAX_EXPERTS\s+(\d+)", header).group(1)) == _lib.MAX_EXPERTS
    for name in ("zrb_ctx_create_mos", "zrb_set_mos_dropout"):
        assert re.search(rf"\b{name}\s*\(", header) and name in _lib.exported_symbols()



def _train_ptb(*args):
    import subprocess
    import sys
    return subprocess.run([sys.executable, os.path.join(ROOT, "tools", "train_ptb.py"), *args], capture_output=True,
                          text=True, timeout=120, cwd=ROOT)


@pytest.mark.parametrize("args,msg", [
    (["--impl", "cudnn", "--experts", "15"], "modes of --impl ours"),
    (["--impl", "cudnn", "--mos_dropout", "0.3"], "modes of --impl ours"),
    (["--mos_dropout", "0.3"], "--mos_dropout needs --experts"),
])
def test_train_ptb_mos_arguments_refused(args, msg):
    r = _train_ptb(*args)
    assert r.returncode != 0 and msg in r.stderr, r.stderr[-2000:]

