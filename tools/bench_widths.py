"""The fused train step of AWD-LSTM's PTB model (DESIGN.md section 18): V = 10000, E = 400, layers 1150-1150-400,
tied, T = 70, B = 20, against a plain-torch cuDNN arm with the same widths, alternated in one process.

    python tools/bench_widths.py [--warmup 20] [--steps 200] [--rounds 3] [--json out.json]

Ours: `Trainer.train_step` (lazy update on and off), CUDA events around each window of steps, plus the per-class split
of one window from zrb_prof_*.  cuDNN: nn.LSTM(400, 1150), nn.LSTM(1150, 1150), nn.LSTM(1150, 400), the tied
projection, cross-entropy (main.py's mean * B), clip_grad_norm_ and SGD in eager torch (cuDNN LSTMs, cuBLAS GEMMs).
No dropout in either arm.  Prints the card name and power limit next to the numbers.
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

V, E, SIZES, T, B, WINIT, LR, CLIP = 10000, 400, (1150, 1150, 400), 70, 20, 0.1, 1.0, 0.25


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


class CudnnAwd(nn.Module):
    """the same widths in plain torch: tied embedding / projection, one nn.LSTM per layer"""

    def __init__(self):
        super().__init__()
        self.embed = nn.Embedding(V, E)
        ins = [E, *SIZES[:-1]]
        self.rnns = nn.ModuleList(nn.LSTM(i, h) for i, h in zip(ins, SIZES))
        self.fc_b = nn.Parameter(torch.zeros(V))
        for p in self.parameters():
            nn.init.uniform_(p, -WINIT, WINIT)

    def forward(self, x, states):
        a = self.embed(x)
        out = []
        for rnn, (h, c) in zip(self.rnns, states):
            a, (h, c) = rnn(a, (h, c))
            out.append((h.detach(), c.detach()))
        return a.reshape(-1, E) @ self.embed.weight.t() + self.fc_b, out


def cudnn_step(model, x, y, states):
    scores, states = model(x, states)
    loss = nn.functional.cross_entropy(scores, y.reshape(-1)) * B
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
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_widths.py measures on a CUDA device; none is available")
    name, power = card()
    print(f"device: {name}, power limit {power}")
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    xs = [torch.randint(0, V, (T, B), generator=g).to(dev) for _ in range(8)]
    ys = [torch.randint(0, V, (T, B), generator=g).to(dev) for _ in range(8)]

    arms = {}
    for lazy in (True, False):
        torch.manual_seed(0)
        m = zaremba_b200.Model(V, SIZES[0], len(SIZES), 0.0, WINIT, tied=True, embed_size=E, layer_sizes=SIZES).to(dev)
        m.train()
        tr = zaremba_b200.Trainer(m, B, T, lazy_update=lazy)
        arms["ours_lazy" if lazy else "ours_strict"] = \
            lambda i, tr=tr: tr.train_step(xs[i % 8], ys[i % 8], LR, CLIP)
    torch.manual_seed(0)
    ref = CudnnAwd().to(dev)
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

    out = dict(device=name, power_limit=power, shape=dict(V=V, E=E, layers=SIZES, T=T, B=B, tied=True),
               warmup=args.warmup, steps=args.steps, ms_per_step=ms,
               tokens_per_s={k: [round(T * B * 1e3 / t, 1) for t in v] for k, v in ms.items()},
               ours_lazy_class_ms_per_step=split)
    for k, v in ms.items():
        print(f"{k:12s} {' '.join(f'{t:.4f}' for t in v)} ms/step  "
              f"{' '.join(f'{T * B * 1e3 / t:.0f}' for t in v)} tokens/s")
    print("ours_lazy per class (ms/step):", ", ".join(f"{c} {t}" for c, t in split.items()))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
