"""Cost of embedding dropout and AR/TAR (DESIGN.md section 17): ms per fused train step of the Small, Medium and Large
configs with both modes off, embedding dropout on (0.1), AR/TAR on (alpha = 2, beta = 1) and both on, under the strict
and the lazy update schedule, alternated in one process.

    python tools/bench_awd_reg.py [--warmup 20] [--steps 300] [--rounds 3] [--json out.json]

Per (config, schedule), four Trainers on the same weights (one per mode) run `warmup` steps each, then `rounds` rounds
of `steps` timed steps per mode, alternating the modes round by round.  Times are CUDA events around each window of steps
on the Trainer's stream.  lr = 0 keeps the weights put; the mode still draws a new mask every step.  Prints the card
name and power limit next to the numbers.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import zaremba_b200  # noqa: E402
from bench_variational import card, window  # noqa: E402
from bench_weight_drop import CONFIGS  # noqa: E402

P_E, AR, TAR = 0.1, 2.0, 1.0
MODES = {"off": (0.0, 0.0, 0.0), "embed": (P_E, 0.0, 0.0), "artar": (0.0, AR, TAR), "both": (P_E, AR, TAR)}


def bench(config, lazy, warmup, steps, rounds):
    V, H, L, T, B, p = CONFIGS[config]
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    xs = [torch.randint(0, V, (T, B), generator=g).to(dev) for _ in range(8)]
    ys = [torch.randint(0, V, (T, B), generator=g).to(dev) for _ in range(8)]
    trainers = {}
    for mode, (pe, ar, tar) in MODES.items():
        torch.manual_seed(0)
        m = zaremba_b200.Model(V, H, L, p, 0.04, embed_dropout=pe).to(dev)
        m.train()
        trainers[mode] = zaremba_b200.Trainer(m, B, T, lazy_update=lazy, ar=ar, tar=tar)
        window(trainers[mode], xs, ys, warmup, lr=0.0)
    ms = {mode: [] for mode in MODES}
    for _ in range(rounds):
        for mode in MODES:
            ms[mode].append(window(trainers[mode], xs, ys, steps, lr=0.0))
    for tr in trainers.values():
        tr.close()
    return dict(config=config, schedule="lazy" if lazy else "strict", H=H, T=T, B=B, embed_dropout=P_E, ar=AR, tar=TAR,
                ms_per_step={mode: v for mode, v in ms.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_awd_reg.py measures on a CUDA device; none is available")
    name, power = card()
    print(f"device: {name}, power limit {power}")
    out = dict(device=name, power_limit=power, warmup=args.warmup, steps=args.steps, results=[])
    for config in ("small", "medium", "large"):
        for lazy in (False, True):
            r = bench(config, lazy, args.warmup, args.steps, args.rounds)
            out["results"].append(r)
            ms = r["ms_per_step"]
            off = min(ms["off"])
            cols = " | ".join(f"{mode} {' '.join(f'{v:.4f}' for v in ms[mode])} (best/off {min(ms[mode]) / off:.4f})"
                              for mode in MODES)
            print(f"{config:6s} {r['schedule']:6s} H={r['H']} ms/step: {cols}", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
