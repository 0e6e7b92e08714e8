"""Layers of unequal width without a GPU: Model's parameters, initialisation and argument checks against a torch stack of
nn.LSTM(In_l, H_l), the fp64 restatement (tests/_model_oracle.py) against torch autograd on such a stack, and the
C declarations of the new entry points."""
import math

import pytest
import torch
from torch import nn

import zaremba_b200
from tests import _model_oracle as O

AWD = dict(tied=True, embed_size=400, layer_sizes=(1150, 1150, 400))


def _torch_stack(V, E, sizes, winit, tied):
    """registration order of Model: embed.W, then each nn.LSTM(In_l, H_l)'s four tensors, fc.W (untied), fc.b"""
    emb = nn.Parameter(torch.empty(V, E))
    lstms = nn.ModuleList(nn.LSTM(([E] + list(sizes))[l], sizes[l]) for l in range(len(sizes)))
    fc_w = emb if tied else nn.Parameter(torch.empty(V, sizes[-1]))
    fc_b = nn.Parameter(torch.empty(V))
    ps = [emb] + [p for m in lstms for p in m.parameters()] + ([] if tied else [fc_w]) + [fc_b]
    for p in ps:
        nn.init.uniform_(p, -winit, winit)
    return emb, lstms, fc_w, fc_b


def test_awd_parameter_names_shapes_and_order():
    m = zaremba_b200.Model(10000, 1150, 3, 0.4, 0.1, **AWD)
    got = [(k, tuple(v.shape)) for k, v in m.named_parameters()]
    want = [("embed.W", (10000, 400))]
    for l, (In, H) in enumerate([(400, 1150), (1150, 1150), (1150, 400)]):
        want += [(f"rnns.{l}.weight_ih_l0", (4 * H, In)), (f"rnns.{l}.weight_hh_l0", (4 * H, H)),
                 (f"rnns.{l}.bias_ih_l0", (4 * H,)), (f"rnns.{l}.bias_hh_l0", (4 * H,))]
    want += [("fc.b", (10000,))]
    assert got == want
    assert m.fc.W is m.embed.W and m.embed_size == 400 and m.layer_sizes == (1150, 1150, 400)
    assert "fc.W" in m.state_dict() and tuple(m.state_dict()["fc.W"].shape) == (10000, 400)
    m2 = zaremba_b200.Model(50, 30, 2, 0.0, 0.1, embed_size=20, layer_sizes=(30, 40))
    assert tuple(m2.fc.W.shape) == (50, 40) and tuple(m2.rnns[1].weight_ih_l0.shape) == (160, 30)


@pytest.mark.parametrize("tied", [False, True])
def test_init_matches_torch_stack_seed_for_seed(tied):
    V, E, sizes, winit = 97, 24, (40, 56, 24), 0.08
    torch.manual_seed(123)
    m = zaremba_b200.Model(V, sizes[0], 3, 0.0, winit, tied=tied, embed_size=E, layer_sizes=sizes)
    after_model = torch.rand(3)
    torch.manual_seed(123)
    emb, lstms, fc_w, fc_b = _torch_stack(V, E, sizes, winit, tied)
    after_stack = torch.rand(3)
    assert torch.equal(after_model, after_stack), "construction consumed the RNG differently"
    assert torch.equal(m.embed.W, emb) and torch.equal(m.fc.W, fc_w) and torch.equal(m.fc.b, fc_b)
    for r, t in zip(m.rnns, lstms):
        for a, b in zip(r.tensors(), t.parameters()):
            assert torch.equal(a, b)


def test_state_dict_round_trip_into_torch_stack_and_back():
    V, E, sizes = 61, 16, (32, 48)
    torch.manual_seed(5)
    m = zaremba_b200.Model(V, 32, 2, 0.0, 0.1, embed_size=E, layer_sizes=sizes)
    sd = m.state_dict()
    emb, lstms, fc_w, fc_b = _torch_stack(V, E, sizes, 0.0, False)
    with torch.no_grad():
        emb.copy_(sd["embed.W"])
        fc_w.copy_(sd["fc.W"])
        fc_b.copy_(sd["fc.b"])
        for l, t in enumerate(lstms):
            t.load_state_dict({k: sd[f"rnns.{l}.{k}"] for k in ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0")})
    m2 = zaremba_b200.model_from_state_dict(sd)
    assert (m2.vocab_size, m2.embed_size, m2.layer_sizes, m2.tied) == (V, E, sizes, False)
    for k, v in m2.state_dict().items():
        assert torch.equal(v, sd[k]), k
    m3 = zaremba_b200.model_from_state_dict(zaremba_b200.Model(V, 40, 2, 0.0, 0.1, tied=True, embed_size=24,
                                                               layer_sizes=(40, 24)).state_dict())
    assert m3.tied and m3.embed_size == 24 and m3.layer_sizes == (40, 24)


def test_state_init_shapes():
    m = zaremba_b200.Model(50, 30, 2, 0.0, 0.1, embed_size=20, layer_sizes=(30, 40))
    assert [tuple(h.shape) for h, _ in m.state_init(3)] == [(1, 3, 30), (1, 3, 40)]


@pytest.mark.parametrize("kw", [
    dict(layer_sizes=(30,)),                                   # wrong length
    dict(layer_sizes=(31, 30)),                                # hidden_size != layer_sizes[0]
    dict(layer_sizes=(30, 0)),
    dict(layer_sizes=(30, 2.5)),
    dict(embed_size=0),
    dict(embed_size=True),
    dict(tied=True, embed_size=20, layer_sizes=(30, 40)),      # E != H_{L-1}
    dict(tied=True, layer_sizes=(30, 40)),                     # E defaults to H = 30
    dict(lstm_type="custom", embed_size=20),
    dict(engine="simt", layer_sizes=(30, 40)),
])
def test_bad_widths_raise(kw):
    with pytest.raises(ValueError):
        zaremba_b200.Model(50, 30, 2, 0.0, 0.1, **kw)


def test_equal_widths_keep_every_mode():
    zaremba_b200.Model(50, 30, 2, 0.0, 0.1, lstm_type="custom", embed_size=30, layer_sizes=(30, 30))
    zaremba_b200.Model(50, 30, 2, 0.0, 0.1, engine="simt", embed_size=30)
    zaremba_b200.Model(50, 30, 2, 0.0, 0.1, tied=True, embed_size=40, layer_sizes=(30, 40))


def test_oracle_matches_torch_autograd_on_lstm_stack():
    """the restatement against nn.LSTM(In_l, H_l) + linear + main.py's loss, float64, tied and untied"""
    V, E, sizes, T, B = 37, 12, (20, 28, 12), 6, 3
    g = torch.Generator().manual_seed(0)
    x = torch.randint(0, V, (T, B), generator=g)
    y = torch.randint(0, V, (T, B), generator=g)
    for tied in (False, True):
        torch.manual_seed(1)
        emb, lstms, fc_w, fc_b = _torch_stack(V, E, sizes, 0.3, tied)
        lstms = lstms.double()
        emb64 = emb.detach().double().requires_grad_(True)
        fcw64 = emb64 if tied else fc_w.detach().double().requires_grad_(True)
        fcb64 = fc_b.detach().double().requires_grad_(True)
        states = [(0.1 * torch.randn(B, H, generator=g, dtype=torch.float64),
                   0.1 * torch.randn(B, H, generator=g, dtype=torch.float64)) for H in sizes]
        out = emb64[x]
        new = []
        for l, t in enumerate(lstms):
            out, (h, c) = t(out, (states[l][0][None], states[l][1][None]))
            new.append((h[0], c[0]))
        scores = out.reshape(T * B, -1) @ fcw64.t() + fcb64
        loss = nn.functional.cross_entropy(scores, y.reshape(-1)) * B
        loss.backward()
        ref = {"embed.W": emb64, "fc.b": fcb64}
        if not tied:
            ref["fc.W"] = fcw64
        for l, t in enumerate(lstms):
            for k, p in t.named_parameters():
                ref[f"rnns.{l}.{k}"] = p
        params = {k: v.detach().clone() for k, v in ref.items()}
        want_loss, norm, grads, after, st, _ = O.train_step(params, x, y, states, len(sizes), tied, 1.0, 0.5)
        assert abs(want_loss - loss.item()) < 1e-12 * max(1, abs(loss.item()))
        assert sorted(grads) == sorted(O.names(len(sizes), tied))
        for k, p in ref.items():
            assert torch.allclose(grads[k], p.grad, rtol=1e-10, atol=1e-13), k
        total = math.sqrt(sum(float((p.grad ** 2).sum()) for p in ref.values()))
        assert abs(norm - total) < 1e-10 * total
        for l in range(len(sizes)):
            assert torch.allclose(st[l][0], new[l][0]) and torch.allclose(st[l][1], new[l][1])


def test_new_entry_points_are_bound():
    from zaremba_b200 import _lib
    assert "zrb_ctx_create_widths" in _lib._SIGNATURES and "zrb_rec_plans_layer" in _lib._SIGNATURES
    hdr = open(_lib.__file__.replace("zaremba_b200/_lib.py", "include/zaremba_b200.h")).read()
    assert "int  zrb_ctx_create_widths(const zrb_config* cfg, const int32_t* widths, zrb_ctx** out);" in hdr
    assert "int  zrb_rec_plans_layer(const zrb_ctx* ctx, int32_t layer, int32_t* h_out);" in hdr


def test_mask_helpers_match_the_equal_width_oracles():
    """at equal widths mode_masks draws exactly the masks of oracle.philox's site_masks and keep_mask"""
    import numpy as np
    from oracle import philox as PH
    L, T, B, H, V = 2, 3, 4, 24, 50
    got = O.mode_masks(O.Modes(seed=9, step=5, p=0.3), [H] * (L + 1), T, B, V).sites
    assert all(np.array_equal(a, b) for a, b in zip(got, PH.site_masks(9, 5, L, T, B, H, 0.3)))
    md = O.Modes(seed=9, step=5, p=0.3, variational=True, p_rec=0.2, wd_seed=11, p_wd=0.4, ed_seed=13, p_e=0.1)
    mk = O.mode_masks(md, [H] * (L + 1), T, B, V)
    for s in range(L + 1):   # variational: the site's first B*H elements at every t
        want = PH.keep_mask(9, 5, s, B * H, 0.3).reshape(B, H)
        assert all(np.array_equal(mk.sites[s][t], want) for t in range(T))
    for l in range(L):
        assert np.array_equal(mk.rec[l], PH.keep_mask(9, 5, L + 1 + l, B * H, 0.2).reshape(B, H))
        assert np.array_equal(mk.wd[l], PH.keep_mask(11, 5, 2 * L + 1 + l, 4 * H * H, 0.4).reshape(4 * H, H))
    assert np.array_equal(mk.ed, PH.keep_mask(13, 5, 3 * L + 1, V, 0.1))
    # unequal widths: each site's stream is over its own width
    mk = O.mode_masks(md, [8, 16, 24], T, B, V)
    sites, rec, wd = mk.sites, mk.rec, mk.wd
    assert [m.shape for m in sites] == [(T, B, 8), (T, B, 16), (T, B, 24)]
    assert np.array_equal(sites[1][2], PH.keep_mask(9, 5, 1, B * 16, 0.3).reshape(B, 16))
    assert [m.shape for m in rec] == [(B, 16), (B, 24)] and [m.shape for m in wd] == [(64, 16), (96, 24)]
    assert np.array_equal(wd[1].reshape(-1), PH.keep_mask(11, 5, 2 * L + 2, 4 * 24 * 24, 0.4))


def _train_ptb(*args):
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    return subprocess.run([sys.executable, os.path.join(root, "tools", "train_ptb.py"), *args], capture_output=True,
                          text=True, timeout=120, cwd=root)


@pytest.mark.parametrize("args,msg", [
    (["--impl", "cudnn", "--layer_sizes", "1150,1150,400"], "modes of --impl ours"),
    (["--impl", "cudnn", "--embed_size", "400"], "modes of --impl ours"),
    (["--layer_sizes", "1150,0"], "positive int"),
    (["--embed_size", "0"], "positive int"),
    (["--tied", "--embed_size", "400", "--layer_sizes", "1150,1150,300"], "--tied needs --embed_size"),
    (["--tied", "--layer_sizes", "1150,400"], "--tied needs --embed_size"),
])
def test_train_ptb_width_arguments_refused(args, msg):
    r = _train_ptb(*args)
    assert r.returncode != 0 and msg in r.stderr, r.stderr[-2000:]


def test_train_ptb_layer_sizes_parse():
    r = _train_ptb("--layer_sizes", "1150,x")
    assert r.returncode == 2 and "--layer_sizes" in r.stderr
