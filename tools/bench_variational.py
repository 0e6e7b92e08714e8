"""Cost of the variational dropout mode (DESIGN.md section 11): the fused train step of the Large and Medium configs
with the mode off and on (recurrent_dropout = dropout, Gal's setting), alternated in one process.

    python tools/bench_variational.py [--warmup 20] [--steps 300] [--rounds 3] [--json out.json]

Per config, two Trainers on the same weights (one per mode) run `warmup` steps each, then `rounds` rounds of `steps`
timed steps per mode, alternating the modes round by round.  Times are CUDA events around each window of steps on the
Trainer's stream.  Prints the card name and power limit next to the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import zaremba_b200  # noqa: E402

CONFIGS = {   # the README's recipes: V, H, L, T, B, p
    "large": (10000, 1500, 2, 35, 20, 0.65),
    "medium": (10000, 650, 2, 35, 20, 0.5),
}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def window(tr, xs, ys, steps, lr=1.0, max_norm=5.0):
    stream = torch.cuda.current_stream()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for i in range(steps):
        tr.train_step(xs[i % len(xs)], ys[i % len(ys)], lr, max_norm)
    b.record(stream)
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
        kw = dict(variational=True) if mode == "on" else {}
        m = zaremba_b200.Model(V, H, L, p, 0.04, **kw).to(dev)
        m.train()
        trainers[mode] = zaremba_b200.Trainer(m, B, T)
        window(trainers[mode], xs, ys, warmup, lr=0.0)
    ms = {"off": [], "on": []}
    for _ in range(rounds):
        for mode in ("off", "on"):
            ms[mode].append(window(trainers[mode], xs, ys, steps, lr=0.0))   # lr 0: the weights stay put
    for tr in trainers.values():
        tr.close()
    return dict(config=config, H=H, T=T, B=B, p=p, ms_per_step_off=ms["off"], ms_per_step_on=ms["on"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_variational.py measures on a CUDA device; none is available")
    name, power = card()
    print(f"device: {name}, power limit {power}")
    out = dict(device=name, power_limit=power, warmup=args.warmup, steps=args.steps, results=[])
    for config in ("large", "medium"):
        r = bench(config, args.warmup, args.steps, args.rounds)
        out["results"].append(r)
        off, on = min(r["ms_per_step_off"]), min(r["ms_per_step_on"])
        print(f"{config:6s} H={r['H']} off {' '.join(f'{v:.4f}' for v in r['ms_per_step_off'])} ms/step | "
              f"on {' '.join(f'{v:.4f}' for v in r['ms_per_step_on'])} ms/step | best on/off {on / off:.4f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
