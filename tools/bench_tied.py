"""Cost of tying the embedding and softmax weights (DESIGN.md section 13): the fused train step of the Small, Medium and
Large configs, tied and untied, with the lazy update off and on, alternated in one process.

    python tools/bench_tied.py [--warmup 20] [--steps 300] [--rounds 3] [--json out.json]

Per config, four Trainers on the same seeded weights ({untied, tied} x {strict, lazy}) run `warmup` steps each, then
`rounds` rounds of `steps` timed steps per variant, alternating the variants round by round.  Times are CUDA events
around each window of steps on the Trainer's stream; the library's launch counter gives launches per step.  A separate
pass under torch.profiler (CUDA activity) sums the device time per step of the tied merge kernels (embed_rows,
embed_first, embed_accum, embed_finish_add) and of the untied embedding-gradient kernels they replace.  Prints the
card name and power limit next to the numbers.
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
from zaremba_b200 import _lib  # noqa: E402

CONFIGS = {   # the README's recipes: V, H, L, T, B, p, winit
    "small": (10000, 200, 2, 20, 20, 0.0, 0.1),
    "medium": (10000, 650, 2, 35, 20, 0.5, 0.05),
    "large": (10000, 1500, 2, 35, 20, 0.65, 0.04),
}
VARIANTS = [("untied", False, False), ("tied", True, False), ("untied_lazy", False, True), ("tied_lazy", True, True)]
EMBED_KERNELS = ("embed_rows", "embed_first", "embed_accum", "embed_finish_add", "embed_finish", "embed_zero_rows",
                 "embed_dropout_bwd", "embed_rows_sumsq", "embed_rows_update")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def window(tr, xs, ys, steps):
    stream = torch.cuda.current_stream()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n0 = _lib.load().zrb_launch_count()
    a.record(stream)
    for i in range(steps):
        tr.train_step(xs[i % len(xs)], ys[i % len(ys)], 0.0, 5.0)   # lr 0: the weights stay put
    b.record(stream)
    b.synchronize()
    return a.elapsed_time(b) / steps, (_lib.load().zrb_launch_count() - n0) / steps


def embed_kernel_us(tr, xs, ys, steps=20):
    """Device time per step (us) of the embedding-gradient kernels, by kernel name, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(steps):
            tr.train_step(xs[i % len(xs)], ys[i % len(ys)], 0.0, 5.0)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        short = next((k for k in EMBED_KERNELS if k + "_kernel" in ev.key), None)
        if short:
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
            out[short] = out.get(short, 0.0) + t / steps
    return out


def bench(config, warmup, steps, rounds):
    V, H, L, T, B, p, winit = CONFIGS[config]
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    xs = [torch.randint(0, V, (T, B), generator=g).to(dev) for _ in range(8)]
    ys = [torch.randint(0, V, (T, B), generator=g).to(dev) for _ in range(8)]
    trainers = {}
    for name, tied, lazy in VARIANTS:
        torch.manual_seed(0)
        m = zaremba_b200.Model(V, H, L, p, winit, tied=tied).to(dev)
        m.train()
        trainers[name] = zaremba_b200.Trainer(m, B, T, lazy_update=lazy)
        window(trainers[name], xs, ys, warmup)
    ms = {name: [] for name, _, _ in VARIANTS}
    launches = {}
    for _ in range(rounds):
        for name, _, _ in VARIANTS:
            t, n = window(trainers[name], xs, ys, steps)
            ms[name].append(t)
            launches[name] = n
    kern = {name: embed_kernel_us(trainers[name], xs, ys) for name in ("untied", "tied")}
    for tr in trainers.values():
        tr.close()
    return dict(config=config, H=H, T=T, B=B, ms_per_step=ms, launches_per_step=launches, embed_kernel_us=kern)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--configs", default="small,medium,large")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tied.py measures on a CUDA device; none is available")
    name, power = card()
    print(f"device: {name}, power limit {power}")
    out = dict(device=name, power_limit=power, warmup=args.warmup, steps=args.steps, results=[])
    for config in args.configs.split(","):
        r = bench(config, args.warmup, args.steps, args.rounds)
        out["results"].append(r)
        for v, _, _ in VARIANTS:
            print(f"{config:6s} {v:12s} {' '.join(f'{t:.4f}' for t in r['ms_per_step'][v])} ms/step, "
                  f"{r['launches_per_step'][v]:.1f} launches/step")
        for v, k in r["embed_kernel_us"].items():
            print(f"{config:6s} {v:12s} embedding-gradient kernels (us/step): "
                  + ", ".join(f"{n} {t:.1f}" for n, t in sorted(k.items())))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
