#!/usr/bin/env python
"""Cost of dynamic evaluation per window (DESIGN.md section 14).

    python tools/bench_dyneval.py [--windows 50] [--rounds 5] [--json out/bench_dyneval.json]

For Small, Medium and Large (V = 10000, L = 2) at (T, B) = (5, 1) and (35, 20), per window, from CUDA events around
`--windows` windows after a warm-up, the variants alternating over `--rounds` rounds (median reported):
  * eval:    the plain eval step (Trainer.eval_step);
  * fused:   the dynamic step with the RMS rule (Trainer.dynamic_eval_step: eval-mode gradient, update, images);
  * eager:   what the drop-in path costs: Model forward in eval mode, the loss in torch, autograd backward, the RMS
             update as torch elementwise ops, and the repack of the fp16 weight images the next forward then does.
Then, in a separate torch.profiler pass, the device time of the fused step's update kernels, and their achieved bandwidth
on the bytes the update must move (computed below from the shapes) against the H100 SXM data sheet's 3.35 TB/s.  The
card's name and power limit are read in the same run.
"""
import argparse, json, os, statistics, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

ap = argparse.ArgumentParser()
ap.add_argument("--configs", default="small,medium,large")
ap.add_argument("--shapes", default="5x1,35x20", help="TxB, comma-separated")
ap.add_argument("--windows", type=int, default=50)
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--json", default=None)
args = ap.parse_args()

import zaremba_b200
from zaremba_b200 import _lib

HIDDEN = {"small": 200, "medium": 650, "large": 1500}
V, L = 10000, 2
HBM_BYTES_PER_S = 3.35e12
LR, LAM, EPS = 1e-4, 0.01, 2e-5
dev = torch.device("cuda", 0)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:            # (reported, not fatal: the timings stand without it)
        q = f"unavailable: {e}"
    return {"name": torch.cuda.get_device_name(0), "power_limit_and_max_sm_clock": q}


def update_bytes(H, plans):
    """Bytes the RMS update must move per window: read theta, g, theta_g, r and write theta (20 B per parameter), plus
    the fp16 images it writes: W_ih's row image [4H, Hp], W_hh's forward and backward recurrent slices (its row image
    when the recurrence takes the per-timestep path) and fc.W's row image [V, Hp]."""
    Hp = (H + 63) // 64 * 64
    P = V * H + L * (2 * 4 * H * H + 2 * 4 * H) + V * H + V
    whh = 4 * H * H * 2 * ((plans["fwd"]["ok"] != 0) + (plans["bwd"]["ok"] != 0)) if plans["fwd"]["ok"] else 4 * H * Hp * 2
    return 20 * P + L * (4 * H * Hp * 2 + whh) + V * Hp * 2


def timed(fn, wins):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for x, y in wins:
        fn(x, y)
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / len(wins)


def eager_step(m, state, tg, r, rbar):
    """One window of the drop-in path: forward, torch loss, autograd backward, the RMS update in torch."""
    params = m.ordered_parameters()

    def step(x, y):
        for p in params:
            p.grad = None
        st = m.detach(state[0])
        scores, st = m(x, st)
        state[0] = st
        loss = -torch.log_softmax(scores, dim=1).gather(1, y.reshape(-1, 1)).mean() * x.shape[1]
        loss.backward()
        with torch.no_grad():
            for p, t, q in zip(params, tg, r):
                u = p.grad / (q + EPS)
                a = (LAM * q / rbar).clamp_(max=1.0)
                p.add_(a * (t - p) - LR * u)
    return step


def update_kernels_us(tr, wins, theta_g, stats):
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for x, y in wins:
            tr.dynamic_eval_step(x, y, theta_g, LR, LAM, stats, EPS)
        torch.cuda.synchronize()
    us = 0.0
    for ev in prof.key_averages():
        if "update_pack" in ev.key or "dyneval_list_kernel" in ev.key:
            us += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
    return us / len(wins)


rows = []
for cfg in args.configs.split(","):
    H = HIDDEN[cfg]
    for shape in args.shapes.split(","):
        T, B = (int(v) for v in shape.split("x"))
        torch.manual_seed(0)
        m = zaremba_b200.Model(V, H, L, 0.5, 1.0 / H ** 0.5).to(dev)
        tr = zaremba_b200.Trainer(m, B, T, data_parallel=False)
        g = torch.Generator(device="cpu").manual_seed(1)
        wins = [(torch.randint(0, V, (T, B), generator=g).to(dev), torch.randint(0, V, (T, B), generator=g).to(dev))
                for _ in range(args.windows)]
        stats = tr.gradient_stats(wins[:4])
        theta_g = tr.flat_p.clone()
        # the drop-in model: the same weights, its own copies of theta_g and r in parameter order
        md = zaremba_b200.Model(V, H, L, 0.5, 1.0 / H ** 0.5).to(dev)
        with torch.no_grad():
            for p, q in zip(md.ordered_parameters(), m.ordered_parameters()):
                p.copy_(q)
        md.eval()
        base = tr.flat_p.data_ptr()
        offs = [((q.data_ptr() - base) // 4, q) for q in m.ordered_parameters()]
        tg = [theta_g[o:o + q.numel()].view_as(q).clone() for o, q in offs]
        rr = [stats.rms[o:o + q.numel()].view_as(q).clone() for o, q in offs]
        state = [md.state_init(B)]
        variants = {
            "eval": lambda x, y: tr.eval_step(x, y),
            "fused": lambda x, y: tr.dynamic_eval_step(x, y, theta_g, LR, LAM, stats, EPS),
            "eager": eager_step(md, state, tg, rr, float(stats.mean)),
        }
        for f in variants.values():
            timed(f, wins[:5])
        ms = {k: [] for k in variants}
        for _ in range(args.rounds):
            for k, f in variants.items():
                tr.flat_p.copy_(theta_g)      # every round adapts from theta_g
                tr.params_changed()
                ms[k].append(timed(f, wins))
        upd_us = update_kernels_us(tr, wins, theta_g, stats)
        nbytes = update_bytes(H, _lib.rec_plans(tr.ctx))
        row = {"config": cfg, "H": H, "T": T, "B": B, **{f"{k}_ms": statistics.median(v) for k, v in ms.items()},
               "update_us": upd_us, "update_bytes": nbytes, "update_GBps": nbytes / (upd_us * 1e-6) / 1e9,
               "update_bound_us": nbytes / HBM_BYTES_PER_S * 1e6,
               "update_share_of_bound": nbytes / HBM_BYTES_PER_S * 1e6 / upd_us}
        rows.append(row)
        print(f"{cfg:6s} T={T:2d} B={B:2d}: eval {row['eval_ms']:.3f} ms, fused dynamic {row['fused_ms']:.3f} ms, "
              f"eager {row['eager_ms']:.3f} ms; update {upd_us:.1f} us for {nbytes / 1e9:.3f} GB = "
              f"{row['update_GBps']:.0f} GB/s ({row['update_share_of_bound']:.2f} of the data-sheet bound)", flush=True)
        del tr, m, md
        torch.cuda.empty_cache()
out = {"card": card(), "lr": LR, "lambda": LAM, "eps": EPS, "rows": rows}
print(json.dumps(out))
if args.json:
    os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
    json.dump(out, open(args.json, "w"), indent=1)
