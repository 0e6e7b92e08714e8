"""The fused train step of the Mixture-of-Softmaxes PTB model (Yang et al. 2018; DESIGN.md section 19): V = 10000,
E = 280, layers 960-960-620, K = 15 experts, tied, T = 70, B = 12, against a plain-torch cuDNN arm of the same model,
alternated in one process.

    python tools/bench_mos.py [--warmup 20] [--steps 100] [--rounds 3] [--json out.json]

Ours: `Trainer.train_step` (lazy update on and off), CUDA events around each window of steps, plus the per-class split
of one window from zrb_prof_* (the head's GEMMs and the LSE pass are in proj_fwd, the mixture-NLL kernel in softmax, the
head's backward GEMMs in proj_bwd).  cuDNN: nn.LSTM(280, 960), nn.LSTM(960, 960), nn.LSTM(960, 620), the MoS head
(Linear + tanh latent, bias-free prior, the tied decoder, the mixture as logsumexp of log-softmaxes), the NLL (main.py's
mean * B), clip_grad_norm_ and SGD in eager torch.  No dropout in either arm.  Prints the card name and power limit and
the bytes the mixture kernels move, computed from the shapes.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import zaremba_b200  # noqa: E402
from zaremba_b200 import _lib  # noqa: E402

V, E, SIZES, K, T, B, WINIT, LR, CLIP = 10000, 280, (960, 960, 620), 15, 70, 12, 0.1, 1.0, 0.25


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


class CudnnMos(nn.Module):
    """the same model in plain torch: tied embedding / decoder, one nn.LSTM per layer, the MoS head"""

    def __init__(self):
        super().__init__()
        self.embed = nn.Embedding(V, E)
        ins = [E, *SIZES[:-1]]
        self.rnns = nn.ModuleList(nn.LSTM(i, h) for i, h in zip(ins, SIZES))
        self.fc_b = nn.Parameter(torch.zeros(V))
        self.prior = nn.Linear(SIZES[-1], K, bias=False)
        self.latent = nn.Linear(SIZES[-1], K * E)
        for p in self.parameters():
            nn.init.uniform_(p, -WINIT, WINIT)

    def forward(self, x, states):
        a = self.embed(x)
        out = []
        for rnn, (h, c) in zip(self.rnns, states):
            a, (h, c) = rnn(a, (h, c))
            out.append((h.detach(), c.detach()))
        h = a.reshape(-1, SIZES[-1])
        z = torch.tanh(self.latent(h)).reshape(-1, E) @ self.embed.weight.t() + self.fc_b
        log_pi = torch.log_softmax(self.prior(h), -1)
        return torch.logsumexp(log_pi[:, :, None] + torch.log_softmax(z, -1).reshape(-1, K, V), 1), out


def cudnn_step(model, x, y, states):
    logp, states = model(x, states)
    loss = nn.functional.nll_loss(logp, y.reshape(-1)) * B
    model.zero_grad(set_to_none=False)
    loss.backward()
    torch.nn.utils.clip_grad_norm_(model.parameters(), CLIP)
    with torch.no_grad():
        for p in model.parameters():
            p.add_(p.grad, alpha=-LR)
    return states


def timed(fn, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(steps):
        fn(i)
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mos.py measures on a CUDA device; none is available")
    name, power = card()
    print(f"device: {name}, power limit {power}")
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    xs = [torch.randint(0, V, (T, B), generator=g).to(dev) for _ in range(8)]
    ys = [torch.randint(0, V, (T, B), generator=g).to(dev) for _ in range(8)]

    arms = {}
    for lazy in (True, False):
        torch.manual_seed(0)
        m = zaremba_b200.Model(V, SIZES[0], len(SIZES), 0.0, WINIT, tied=True, embed_size=E, layer_sizes=SIZES,
                               experts=K).to(dev)
        m.train()
        tr = zaremba_b200.Trainer(m, B, T, lazy_update=lazy)
        arms["ours_lazy" if lazy else "ours_strict"] = \
            lambda i, tr=tr: tr.train_step(xs[i % 8], ys[i % 8], LR, CLIP)
    torch.manual_seed(0)
    ref = CudnnMos().to(dev)
    ref_states = [[(torch.zeros(1, B, h, device=dev), torch.zeros(1, B, h, device=dev)) for h in SIZES]]

    def ref_fn(i):
        ref_states[0] = cudnn_step(ref, xs[i % 8], ys[i % 8], ref_states[0])
    arms["cudnn"] = ref_fn

    for fn in arms.values():
        timed(fn, args.warmup)
    ms = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, fn in arms.items():
            ms[k].append(timed(fn, args.steps))

    # per-class split of the lazy arm (a separate window: the event brackets add host work)
    tr = arms["ours_lazy"].__defaults__[0]
    lib = _lib.load()
    _lib.check(lib.zrb_prof_enable(tr.ctx, 1))
    timed(arms["ours_lazy"], 50)
    cls_ms = (C.c_float * 16)()
    cls_n = (C.c_int64 * 16)()
    _lib.check(lib.zrb_prof_read(tr.ctx, cls_ms, cls_n))
    _lib.check(lib.zrb_prof_enable(tr.ctx, 0))
    split = {c: round(cls_ms[i] / 50, 4) for i, c in enumerate(_lib.PROF_CLASSES)}

    # bytes from shapes: the LSE pass reads the N*K logits rows once (fp32); the mixture-NLL kernel reads them again and
    # writes the fp16 gradient rows (pitch pad64(V))
    NK, Vp = T * B * K, (V + 63) // 64 * 64
    mix_bytes = dict(lse=NK * V * 4, nll_grad=NK * V * 4 + NK * Vp * 2)
    ws = lib.zrb_ctx_workspace_bytes(tr.ctx)
    out = dict(device=name, power_limit=power, shape=dict(V=V, E=E, layers=SIZES, K=K, T=T, B=B, tied=True),
               warmup=args.warmup, steps=args.steps, ms_per_step=ms,
               tokens_per_s={k: [round(T * B * 1e3 / t, 1) for t in v] for k, v in ms.items()},
               ours_lazy_class_ms_per_step=split, mixture_bytes=mix_bytes, workspace_bytes=ws)
    for k, v in ms.items():
        print(f"{k:12s} {' '.join(f'{t:.4f}' for t in v)} ms/step  "
              f"{' '.join(f'{T * B * 1e3 / t:.0f}' for t in v)} tokens/s")
    print("ours_lazy per class (ms/step):", ", ".join(f"{c} {t}" for c, t in split.items()))
    print(f"mixture kernels' bytes per step: LSE {mix_bytes['lse'] / 1e6:.0f} MB, NLL + gradient "
          f"{mix_bytes['nll_grad'] / 1e6:.0f} MB; softmax class at {split['softmax']} ms = "
          f"{mix_bytes['nll_grad'] / (split['softmax'] * 1e-3) / 1e12:.2f} TB/s; context workspace {ws / 1e9:.2f} GB")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
