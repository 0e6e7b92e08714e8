"""Cost of zoneout (DESIGN.md section 20): ms per fused train step of the Medium and Large configs with the mode off and on
(zoneout_cell = 0.5, zoneout_hidden = 0.05, the paper's LSTM rates), alternated in one process, and a plain-torch arm: an
`nn.LSTMCell` loop with zoneout (the way to get zoneout without this library, since cuDNN's fused LSTM keeps c inside),
with autograd, clip_grad_norm_ and SGD.

    python tools/bench_zoneout.py [--warmup 20] [--steps 200] [--rounds 3] [--torch_steps 20] [--json out.json]

Times are CUDA events around each window of steps on the stream the work runs on.  lr = 0 keeps the weights put; the
mode still draws its flags every step.  Prints the card name and power limit next to the numbers.
"""
import argparse
import json
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import zaremba_b200  # noqa: E402
from bench_variational import card, window  # noqa: E402

CONFIGS = {   # the README's recipes: V, H, L, T, B, p
    "medium": (10000, 650, 2, 35, 20, 0.5),
    "large": (10000, 1500, 2, 35, 20, 0.65),
}
Z_C, Z_H = 0.5, 0.05


class TorchZoneout(nn.Module):
    """the realistic alternative: Zaremba's model with an LSTMCell loop per layer and Krueger et al.'s zoneout"""

    def __init__(self, V, H, L, p):
        super().__init__()
        self.embed = nn.Embedding(V, H)
        self.cells = nn.ModuleList(nn.LSTMCell(H, H) for _ in range(L))
        self.fc = nn.Linear(H, V)
        self.drop = nn.Dropout(p)

    def forward(self, x, states):
        a = self.drop(self.embed(x))
        out = []
        for l, cell in enumerate(self.cells):
            h, c = states[l]
            ys = []
            for t in range(a.shape[0]):
                h2, c2 = cell(a[t], (h, c))
                zc = (torch.rand_like(c) < Z_C).to(c.dtype)
                zh = (torch.rand_like(h) < Z_H).to(h.dtype)
                c = zc * c + (1 - zc) * c2
                h = zh * h + (1 - zh) * h2
                ys.append(h)
            out.append((h.detach(), c.detach()))
            a = self.drop(torch.stack(ys))
        return self.fc(a.reshape(-1, a.shape[-1])), out


def torch_arm(config, warmup, steps):
    V, H, L, T, B, p = CONFIGS[config]
    dev = torch.device("cuda:0")
    m = TorchZoneout(V, H, L, p).to(dev).train()
    opt = torch.optim.SGD(m.parameters(), lr=0.0)
    g = torch.Generator().manual_seed(0)
    x = torch.randint(0, V, (T, B), generator=g).to(dev)
    y = torch.randint(0, V, (T, B), generator=g).to(dev)
    states = [(torch.zeros(B, H, device=dev), torch.zeros(B, H, device=dev)) for _ in range(L)]

    def step():
        nonlocal states
        opt.zero_grad(set_to_none=True)
        scores, states = m(x, states)
        nn.functional.cross_entropy(scores, y.reshape(-1)).backward()
        nn.utils.clip_grad_norm_(m.parameters(), 5.0)
        opt.step()

    for _ in range(warmup):
        step()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        step()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def bench(config, warmup, steps, rounds):
    V, H, L, T, B, p = CONFIGS[config]
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    xs = [torch.randint(0, V, (T, B), generator=g).to(dev) for _ in range(8)]
    ys = [torch.randint(0, V, (T, B), generator=g).to(dev) for _ in range(8)]
    trainers = {}
    for mode in ("off", "on"):
        torch.manual_seed(0)
        z = (Z_C, Z_H) if mode == "on" else (0.0, 0.0)
        m = zaremba_b200.Model(V, H, L, p, 0.04, zoneout_cell=z[0], zoneout_hidden=z[1]).to(dev)
        m.train()
        trainers[mode] = zaremba_b200.Trainer(m, B, T)
        window(trainers[mode], xs, ys, warmup, lr=0.0)
    ms = {"off": [], "on": []}
    for _ in range(rounds):
        for mode in ("off", "on"):
            ms[mode].append(window(trainers[mode], xs, ys, steps, lr=0.0))
    for tr in trainers.values():
        tr.close()
    return dict(config=config, H=H, T=T, B=B, zoneout_cell=Z_C, zoneout_hidden=Z_H, ms_per_step_off=ms["off"],
                ms_per_step_on=ms["on"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--torch_steps", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_zoneout.py measures on a CUDA device; none is available")
    name, power = card()
    print(f"device: {name}, power limit {power}")
    out = dict(device=name, power_limit=power, warmup=args.warmup, steps=args.steps, results=[])
    for config in CONFIGS:
        r = bench(config, args.warmup, args.steps, args.rounds)
        r["ms_per_step_torch"] = torch_arm(config, min(args.warmup, 5), args.torch_steps)
        out["results"].append(r)
        off, on = min(r["ms_per_step_off"]), min(r["ms_per_step_on"])
        print(f"{config:6s} H={r['H']} off {' '.join(f'{v:.4f}' for v in r['ms_per_step_off'])} ms/step | on "
              f"{' '.join(f'{v:.4f}' for v in r['ms_per_step_on'])} ms/step | best on/off {on / off:.4f} | torch "
              f"LSTMCell arm {r['ms_per_step_torch']:.3f} ms/step ({r['ms_per_step_torch'] / on:.1f}x the fused step)",
              flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
