#!/usr/bin/env python
"""Cost of the neural cache per evaluation window (DESIGN.md section 12).

    python tools/bench_cache.py [--windows 50] [--rounds 5] [--json out/bench_cache.json]

For Small, Medium and Large (V = 10000, L = 2, T = 35), B in {1, 20} and W in {100, 500, 2000}:
  * the eval step's time per window without and with the cache: CUDA events around `--windows` windows, after a
    warm-up, the two variants alternating over `--rounds` rounds (median reported);
  * the device time of the cache's own launches (append, attend, combine) from torch.profiler in a separate pass,
    and the attend kernel's bandwidth on key bytes against the bound B * (W + T) * Hp * 2 / 3.35 TB/s (the H100 SXM
    data sheet's HBM3 bandwidth);
  * the card's name and power limit, read in the same run.
"""
import argparse, json, os, statistics, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

ap = argparse.ArgumentParser()
ap.add_argument("--configs", default="small,medium,large")
ap.add_argument("--batches", default="1,20")
ap.add_argument("--sizes", default="100,500,2000")
ap.add_argument("--windows", type=int, default=50)
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--json", default=None)
args = ap.parse_args()

import zaremba_b200

HIDDEN = {"small": 200, "medium": 650, "large": 1500}
V, L, T = 10000, 2, 35
HBM_BYTES_PER_S = 3.35e12
dev = torch.device("cuda", 0)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:            # (reported, not fatal: the timings stand without it)
        q = f"unavailable: {e}"
    return {"name": torch.cuda.get_device_name(0), "power_limit_and_max_sm_clock": q}


def timed(tr, wins, cache, theta, lam):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for x, y in wins:
        if cache is None:
            tr.eval_step(x, y)
        else:
            tr.eval_step(x, y, cache=cache, theta=theta, lam=lam)
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / len(wins)


def cache_kernel_us(tr, wins, cache):
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for x, y in wins:
            tr.eval_step(x, y, cache=cache, theta=0.3, lam=0.1)
        torch.cuda.synchronize()
    us = {"append": 0.0, "attend": 0.0, "combine": 0.0}
    for ev in prof.key_averages():
        for k in us:
            if f"cache_{k}_kernel" in ev.key:
                us[k] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
    return {k: v / len(wins) for k, v in us.items()}


rows = []
for cfg in args.configs.split(","):
    H = HIDDEN[cfg]
    Hp = (H + 63) // 64 * 64
    for B in [int(b) for b in args.batches.split(",")]:
        torch.manual_seed(0)
        model = zaremba_b200.Model(V, H, L, 0.0, 1.0 / H ** 0.5).to(dev)
        tr = zaremba_b200.Trainer(model, B, T)
        g = torch.Generator(device="cpu").manual_seed(1)
        wins = [(torch.randint(0, V, (T, B), generator=g).to(dev), torch.randint(0, V, (T, B), generator=g).to(dev))
                for _ in range(args.windows)]
        for W in [int(w) for w in args.sizes.split(",")]:
            cache = zaremba_b200.NeuralCache(H, B, W, T)
            timed(tr, wins, None, 0, 0); timed(tr, wins, cache, 0.3, 0.1)      # warm-up; the cache fills to W
            plain, cached = [], []
            for _ in range(args.rounds):
                plain.append(timed(tr, wins, None, 0, 0))
                cached.append(timed(tr, wins, cache, 0.3, 0.1))
            k_us = cache_kernel_us(tr, wins, cache)
            key_bytes = B * (W + T) * Hp * 2
            bound_us = key_bytes / HBM_BYTES_PER_S * 1e6
            row = {"config": cfg, "H": H, "B": B, "W": W, "eval_ms": statistics.median(plain),
                   "eval_cache_ms": statistics.median(cached), "cache_kernels_us": k_us,
                   "key_bytes": key_bytes, "key_bound_us": bound_us,
                   "attend_key_GBps": key_bytes / (k_us["attend"] * 1e-6) / 1e9 if k_us["attend"] else None,
                   "attend_share_of_bound": bound_us / k_us["attend"] if k_us["attend"] else None}
            rows.append(row)
            print(f"{cfg:6s} B={B:2d} W={W:4d}: eval {row['eval_ms']:.3f} ms, with cache {row['eval_cache_ms']:.3f} ms; "
                  f"append {k_us['append']:.1f} attend {k_us['attend']:.1f} combine {k_us['combine']:.1f} us; "
                  f"key bound {bound_us:.1f} us ({row['attend_share_of_bound'] or 0:.2f} of it)", flush=True)
            cache.close()
        del tr, model
        torch.cuda.empty_cache()
out = {"card": card(), "rows": rows}
print(json.dumps(out))
if args.json:
    os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
    json.dump(out, open(args.json, "w"), indent=1)
