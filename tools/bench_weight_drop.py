"""Cost of the weight-dropped LSTM (DESIGN.md section 15): ms per fused train step of the Small, Medium and Large configs
with the mode off and on (weight_drop = 0.5), under the strict and the lazy update schedule, alternated in one process.

    python tools/bench_weight_drop.py [--warmup 20] [--steps 300] [--rounds 3] [--json out.json]

Per (config, schedule), two Trainers on the same weights (one per mode) run `warmup` steps each, then `rounds` rounds of
`steps` timed steps per mode, alternating the modes round by round.  Times are CUDA events around each window of steps
on the Trainer's stream.  lr = 0 keeps the weights put; the mode still draws a new mask and packs new images every step.
Prints the card name and power limit next to the numbers.
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

CONFIGS = {   # the README's recipes: V, H, L, T, B, p
    "small": (10000, 200, 2, 20, 20, 0.0),
    "medium": (10000, 650, 2, 35, 20, 0.5),
    "large": (10000, 1500, 2, 35, 20, 0.65),
}
P_WD = 0.5


def bench(config, lazy, warmup, steps, rounds):
    V, H, L, T, B, p = CONFIGS[config]
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    xs = [torch.randint(0, V, (T, B), generator=g).to(dev) for _ in range(8)]
    ys = [torch.randint(0, V, (T, B), generator=g).to(dev) for _ in range(8)]
    trainers = {}
    for mode in ("off", "on"):
        torch.manual_seed(0)
        m = zaremba_b200.Model(V, H, L, p, 0.04, weight_drop=P_WD if mode == "on" else 0.0).to(dev)
        m.train()
        trainers[mode] = zaremba_b200.Trainer(m, B, T, lazy_update=lazy)
        window(trainers[mode], xs, ys, warmup, lr=0.0)
    ms = {"off": [], "on": []}
    for _ in range(rounds):
        for mode in ("off", "on"):
            ms[mode].append(window(trainers[mode], xs, ys, steps, lr=0.0))
    for tr in trainers.values():
        tr.close()
    return dict(config=config, schedule="lazy" if lazy else "strict", H=H, T=T, B=B, weight_drop=P_WD,
                ms_per_step_off=ms["off"], ms_per_step_on=ms["on"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_weight_drop.py measures on a CUDA device; none is available")
    name, power = card()
    print(f"device: {name}, power limit {power}")
    out = dict(device=name, power_limit=power, warmup=args.warmup, steps=args.steps, results=[])
    for config in ("small", "medium", "large"):
        for lazy in (False, True):
            r = bench(config, lazy, args.warmup, args.steps, args.rounds)
            out["results"].append(r)
            off, on = min(r["ms_per_step_off"]), min(r["ms_per_step_on"])
            print(f"{config:6s} {r['schedule']:6s} H={r['H']} off {' '.join(f'{v:.4f}' for v in r['ms_per_step_off'])} "
                  f"ms/step | on {' '.join(f'{v:.4f}' for v in r['ms_per_step_on'])} ms/step | best on/off {on / off:.4f}",
                  flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
