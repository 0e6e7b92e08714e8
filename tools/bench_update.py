#!/usr/bin/env python
"""Where the end-of-step weight update spends its time (DESIGN.md section 4.4).

    python tools/bench_update.py --out <dir> [--configs small,medium,large] [--steps 10] [--warmup 5]

For each config, fused train steps on the strict schedule (Trainer(lazy_update=False): every update at the end of its
own step) run under torch.profiler with CUDA activities, in a pass of its own after a warm-up.  In each profiled step
the contiguous run of update-phase launches that ends with the list update of the biases (clip_sgd_update_kernel) is
picked out of the trace and every launch of it gets a role:

  update_pack_kernel        W_ih of each layer (row image), then fc.W (row image)
  update_pack_whh_kernel    W_hh of each layer (forward and backward recurrent slices, or its row image when the
                            recurrence takes the per-timestep path)
  the small launches        first-occurrence table of the window's tokens (memset + embed_first_kernel), the embedding
                            rows' sum of squares, the partials memset, the biases' sum of squares, the norm, the
                            embedding rows update and the biases' update (sgd_apply)

Per role: device time per step, the bytes it must move (computed below from the shapes, the window's tokens and the
recurrence plans), and the achieved GB/s.  The ceiling is measured in the same process: a device-to-device copy of
1 GiB (torch copy_), counted as read plus write bytes.  The GPU name, power limit and SM clocks are read in the same
run.  Writes bench_update.json and the profiler tables to --out.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

CONFIGS = {  # name: H, T, B, dropout, winit (bench.py CONFIGS)
    "small": (200, 20, 20, 0.0, 0.1), "medium": (650, 35, 20, 0.5, 0.05), "large": (1500, 35, 20, 0.65, 0.04)}
V, L = 10000, 2
N_NORM_PARTIALS = 148 * 8 + 1024          # optim.cu kNormBlocks + kernels.h kNormExtra


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        row = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:            # (reported, not fatal: the timings stand without it)
        row = f"unavailable: {e}"
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q, "value": row}


def copy_ceiling(nbytes=1 << 30, reps=20):
    """GB/s of a device-to-device torch copy_ of `nbytes`, counted as read + write."""
    src = torch.empty(nbytes // 4, dtype=torch.float32, device="cuda").uniform_()
    dst = torch.empty_like(src)
    for _ in range(3):
        dst.copy_(src)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        dst.copy_(src)
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / reps
    del src, dst
    torch.cuda.empty_cache()
    return {"bytes_per_copy": nbytes, "ms": ms, "GBps": 2 * nbytes / (ms * 1e-3) / 1e9}


def role_bytes(H, T, B, plans, uniq):
    """Bytes each launch of the strict end-of-step update must move (keep_clipped off: g is read, not written back).
    uniq: distinct tokens of the window (the embedding rows the norm and the update touch)."""
    N = T * B
    mat = 4 * H * H          # (the row images are written in their H real columns only, not the pad)
    fwd_ok, bwd_ok = bool(plans["fwd"]["ok"]), bool(plans["bwd"]["ok"])
    # W_hh: a slice image per persistent plan, and the row image unless both plans are persistent (engine_tc.cu)
    whh_images = 2 * mat * (int(fwd_ok) + int(bwd_ok) + int(not (fwd_ok and bwd_ok)))
    biases = L * 8 * H + V
    return {
        "W_ih update_pack": mat * 12 + mat * 2,
        "W_hh update_pack_whh": mat * 12 + whh_images,
        "fc.W update_pack": V * H * 12 + V * H * 2,
        "memset first table": V * 4,
        "embed_first_kernel": N * 8 + N * 4,
        "embed_rows_sumsq": N * 8 + N * 4 + uniq * H * 4,
        "memset partials": N_NORM_PARTIALS * 4,
        "sumsq (biases)": biases * 4,
        "norm_finalize": None,    # reads the partials and the wgrad epilogue slots: a few tens of KB
        "embed_rows_update": N * 8 + N * 4 + uniq * H * 12,
        "sgd_apply (biases)": biases * 12,
    }


def role_names(events):
    """Roles of one step's update-phase launches, in launch order."""
    roles, seen = [], {}
    for name in events:
        k = seen.get(name, 0)
        seen[name] = k + 1
        if "update_pack_whh_kernel" in name:
            roles.append("W_hh update_pack_whh")
        elif "update_pack_kernel" in name:
            roles.append("fc.W update_pack" if k == L else "W_ih update_pack")
        elif name.startswith("Memset"):
            roles.append("memset first table" if k == 0 else "memset partials" if k == 1 else f"memset #{k}")
        elif "embed_first_kernel" in name:
            roles.append("embed_first_kernel")
        elif "embed_rows_sumsq" in name:
            roles.append("embed_rows_sumsq")
        elif "sumsq_kernel" in name:
            roles.append("sumsq (biases)")
        elif "norm_finalize" in name:
            roles.append("norm_finalize")
        elif "embed_rows_update" in name:
            roles.append("embed_rows_update")
        elif "clip_sgd_update_kernel" in name:
            roles.append("sgd_apply (biases)")
        else:
            roles.append(name)
    return roles


PHASE = ("Memset", "embed_first_kernel", "embed_rows_sumsq", "sumsq_kernel", "norm_finalize", "embed_rows_update",
         "update_pack_kernel", "update_pack_whh_kernel", "clip_sgd_update_kernel")


def in_phase(name):
    return any(name.startswith(p) or p in name for p in PHASE)


def run_config(cfg, args, out_dir):
    import zaremba_b200
    from zaremba_b200 import _lib
    from torch.profiler import profile, ProfilerActivity
    H, T, B, p, winit = CONFIGS[cfg]
    dev = torch.device("cuda", 0)
    torch.manual_seed(1)
    model = zaremba_b200.Model(V, H, L, p, winit).to(dev)
    model.train()
    tr = zaremba_b200.Trainer(model, B, T, lazy_update=False)
    g = torch.Generator().manual_seed(2)
    n = args.warmup + args.steps
    data = torch.randint(0, V, (B, T * n + 1), generator=g, dtype=torch.int64)
    wins = [(data[:, i * T:(i + 1) * T].t().contiguous(), data[:, i * T + 1:(i + 1) * T + 1].t().contiguous())
            for i in range(n)]
    uniq = sum(int(torch.unique(x).numel()) for x, _ in wins[args.warmup:]) / args.steps
    wins = [(x.to(dev), y.to(dev)) for x, y in wins]
    for x, y in wins[:args.warmup]:
        tr.train_step(x, y, 1.0, 5.0)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for x, y in wins[args.warmup:]:
            tr.train_step(x, y, 1.0, 5.0)
        torch.cuda.synchronize()
    table = prof.key_averages().table(sort_by="self_device_time_total", row_limit=60)
    with open(os.path.join(out_dir, f"bench_update_{cfg}_profile.txt"), "w") as f:
        f.write(table)
    evs = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                 key=lambda e: e.time_range.start)
    names = [e.name for e in evs]
    ends = [i for i, nm in enumerate(names) if "clip_sgd_update_kernel" in nm]
    per_role, phases = {}, []
    for end in ends:
        start = end
        while start > 0 and in_phase(names[start - 1]):
            start -= 1
        phase = evs[start:end + 1]
        phases.append([e.name for e in phase])
        for role, e in zip(role_names([e.name for e in phase]), phase):
            per_role.setdefault(role, []).append(e.time_range.elapsed_us())
    plans = _lib.rec_plans(tr.ctx)
    nbytes = role_bytes(H, T, B, plans, uniq)
    steps = len(ends)
    rows = []
    for role, us in per_role.items():
        launches = len(us) / steps
        us_step = sum(us) / steps
        b = nbytes.get(role)
        b_step = b * launches if b is not None else None
        rows.append({"role": role, "launches_per_step": launches, "us_per_step": us_step,
                     "us_per_launch": us_step / launches, "bytes_per_step": b_step,
                     "GBps": b_step / (us_step * 1e-6) / 1e9 if b_step else None})
    total_us = sum(r["us_per_step"] for r in rows)
    del tr, model
    torch.cuda.empty_cache()
    return {"config": cfg, "H": H, "T": T, "B": B, "plans": plans, "profiled_steps": steps,
            "unique_tokens_per_window": uniq, "phase_launch_names": phases[0] if phases else [],
            "phase_us_per_step": total_us, "roles": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--configs", default="small,medium,large")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_update.py needs a CUDA device")
    os.makedirs(args.out, exist_ok=True)
    res = {"card": card(), "copy_ceiling": copy_ceiling(), "configs": []}
    ceil = res["copy_ceiling"]["GBps"]
    print(f"copy ceiling {ceil:.0f} GB/s ({res['card']['value']})", flush=True)
    for cfg in args.configs.split(","):
        r = run_config(cfg, args, args.out)
        for row in r["roles"]:
            row["of_copy"] = row["GBps"] / ceil if row["GBps"] else None
            gbs = f"{row['GBps']:7.0f} GB/s ({row['of_copy']:.2f} of copy)" if row["GBps"] else ""
            print(f"{cfg:6s} {row['role']:22s} x{row['launches_per_step']:.0f} {row['us_per_step']:8.1f} us/step {gbs}",
                  flush=True)
        print(f"{cfg:6s} update phase {r['phase_us_per_step']:.1f} us/step (sum of launches)", flush=True)
        res["configs"].append(r)
    res["card_after"] = card()
    with open(os.path.join(args.out, "bench_update.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
