"""Cost of iterate averaging (NT-ASGD, DESIGN.md section 16) at the Small, Medium and Large configs.

    python tools/bench_asgd.py [--warmup 20] [--steps 300] [--rounds 3] [--json out.json]

1. ms per fused train step with averaging off and on, under the strict and the lazy update schedule: two Trainers on
   the same weights (one per mode) run `warmup` steps each, then `rounds` rounds of `steps` timed steps per mode,
   alternating the modes round by round (CUDA events on the Trainer's stream).  lr = 0 keeps the weights put; the
   averaged update streams the average all the same.
2. ms per zrb_swap_average (the mean of 2 * 50 swaps: in and back).
3. Under torch.profiler, in a run of its own: the GPU time of the new kernels in one averaged step and one swap, their
   bytes over that time, against a device-to-device copy of the flat parameter buffer (read + write) timed the same way.
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
from bench_weight_drop import CONFIGS  # noqa: E402

NEW_KERNELS = ("AvgRule", "SwapRule", "sgd_avg_list_kernel", "swap_list_kernel")


def _pair(config, lazy, warmup):
    V, H, L, T, B, p = CONFIGS[config]
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    xs = [torch.randperm(V, generator=g)[:T * B].view(T, B).to(dev) for _ in range(8)]
    ys = [torch.randint(0, V, (T, B), generator=g).to(dev) for _ in range(8)]
    trainers = {}
    for mode in ("off", "on"):
        torch.manual_seed(0)
        m = zaremba_b200.Model(V, H, L, p, 0.04).to(dev)
        m.train()
        trainers[mode] = zaremba_b200.Trainer(m, B, T, lazy_update=lazy)
        if mode == "on":
            trainers[mode].start_averaging()
        window(trainers[mode], xs, ys, warmup, lr=0.0)
    return trainers, xs, ys


def _swap_ms(tr, n=50):
    tr.flush()
    s = torch.cuda.current_stream()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(s)
    for _ in range(n):
        with tr.averaged_weights():
            pass
    b.record(s)
    b.synchronize()
    return a.elapsed_time(b) / (2 * n)


def _profile(tr, xs, ys):
    """{kernel name: us} of one averaged strict step and one swap in and back, and the us of a flat D2D copy."""
    from torch.profiler import ProfilerActivity, profile
    tr.flush()
    dst = torch.empty_like(tr.flat_p)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        tr.train_step(xs[0], ys[0], 0.0, 0.25)
        tr.flush()
        with tr.averaged_weights():
            pass
        dst.copy_(tr.flat_p)
        torch.cuda.synchronize()
    out, copy_us = {}, 0.0
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if any(k in e.key for k in NEW_KERNELS):
            out[e.key[:120]] = out.get(e.key[:120], 0.0) + t
        elif "Memcpy DtoD" in e.key or "copy" in e.key.lower() and "elementwise" in e.key.lower():
            copy_us += t
    return out, copy_us


def bench(config, warmup, steps, rounds):
    rows = []
    for lazy in (False, True):
        trainers, xs, ys = _pair(config, lazy, warmup)
        ms = {"off": [], "on": []}
        for _ in range(rounds):
            for mode in ("off", "on"):
                ms[mode].append(window(trainers[mode], xs, ys, steps, lr=0.0))
        row = dict(config=config, schedule="lazy" if lazy else "strict", ms_per_step_off=ms["off"],
                   ms_per_step_on=ms["on"])
        if not lazy:
            tr = trainers["on"]
            row["ms_per_swap"] = _swap_ms(tr)
            kern, copy_us = _profile(tr, xs, ys)
            n = tr.flat_p.numel()
            row["kernels_us"] = kern
            row["copy_us"] = copy_us
            row["copy_GBps"] = 8 * n / copy_us / 1e3 if copy_us else None
            # bytes of the averaged step's new kernels: the update's 16 B per element (+ images) plus 8 B of the
            # average; the dense embedding pass 12 B per element.  The swap: 16 B per element (+ images).
            row["flat_elements"] = n
        rows.append(row)
        for t in trainers.values():
            t.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_asgd.py measures on a CUDA device; none is available")
    name, power = card()
    print(f"device: {name}, power limit {power}")
    out = dict(device=name, power_limit=power, warmup=args.warmup, steps=args.steps, results=[])
    for config in ("small", "medium", "large"):
        for r in bench(config, args.warmup, args.steps, args.rounds):
            out["results"].append(r)
            off, on = min(r["ms_per_step_off"]), min(r["ms_per_step_on"])
            line = (f"{config:6s} {r['schedule']:6s} off {' '.join(f'{v:.4f}' for v in r['ms_per_step_off'])} ms/step | "
                    f"on {' '.join(f'{v:.4f}' for v in r['ms_per_step_on'])} ms/step | best on/off {on / off:.4f}")
            if "ms_per_swap" in r:
                line += f" | swap {r['ms_per_swap']:.4f} ms | flat copy {r['copy_us']:.1f} us ({r['copy_GBps']:.0f} GB/s)"
            print(line, flush=True)
            for k, v in sorted(r.get("kernels_us", {}).items()):
                print(f"    {v:9.1f} us  {k}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
