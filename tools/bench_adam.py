"""Cost of Adam in the fused train step (DESIGN.md section 21) at the Small, Medium and Large configs.

    python tools/bench_adam.py [--warmup 20] [--steps 300] [--rounds 3] [--json out.json]

1. ms per fused train step with SGD and with Adam, under the strict and the lazy update schedule: two Trainers on the
   same weights (one per optimizer) run `warmup` steps each, then `rounds` rounds of `steps` timed steps per optimizer,
   alternating round by round (CUDA events on the Trainer's stream).  lr = 0 keeps the weights put; both updates
   stream all their bytes all the same.
2. The update class (zrb_prof, "clip_sgd": the clip norm and the update kernels) of the strict arms in a window of its
   own, with the bytes each update must move computed from the shapes, and the rate that gives.
3. A plain-torch arm: the cuDNN nn.LSTM model of oracle/torch_port.py, clip_grad_norm_ and torch.optim.Adam(fused=True).
Prints the card name and power limit next to the numbers.
"""
import argparse
import ctypes as C
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import zaremba_b200  # noqa: E402
from zaremba_b200 import _lib  # noqa: E402
from bench_variational import card, window  # noqa: E402
from bench_weight_drop import CONFIGS  # noqa: E402

WINDOWS = 8


def _data(config):
    V, H, L, T, B, p = CONFIGS[config]
    g = torch.Generator().manual_seed(0)
    xs = [torch.randperm(V, generator=g)[:T * B].view(T, B).cuda() for _ in range(WINDOWS)]
    ys = [torch.randint(0, V, (T, B), generator=g).cuda() for _ in range(WINDOWS)]
    return xs, ys


def _trainers(config, lazy, xs, ys, warmup):
    V, H, L, T, B, p = CONFIGS[config]
    out = {}
    for opt in ("sgd", "adam"):
        torch.manual_seed(0)
        m = zaremba_b200.Model(V, H, L, p, 0.04).cuda()
        m.train()
        out[opt] = zaremba_b200.Trainer(m, B, T, lazy_update=lazy, optimizer=opt)
        window(out[opt], xs, ys, warmup, lr=0.0)
    return out


def _update_ms(tr, xs, ys, n=50):
    """ms per step of the update class (clip norm + update kernels), strict schedule"""
    lib = _lib.load()
    _lib.check(lib.zrb_prof_enable(tr.ctx, 1))
    window(tr, xs, ys, n, lr=0.0)
    ms = (C.c_float * 16)()
    cnt = (C.c_int64 * 16)()
    _lib.check(lib.zrb_prof_read(tr.ctx, ms, cnt))
    _lib.check(lib.zrb_prof_enable(tr.ctx, 0))
    return ms[_lib.PROF_CLASSES.index("clip_sgd")] / n


def update_bytes(config):
    """Bytes the update kernels of one strict step must move (the Trainer's defaults: rows-only embedding under SGD,
    no g' store), from the shapes.  Per element: SGD reads g, p and writes p (12 B); Adam reads g, p, m, v and writes
    p, m, v (28 B).  Plus the fp16 images: 2 B per W_ih / fc.W element, 4 B per W_hh element (forward and backward
    slices).  The SGD embedding touches the window's T*B rows only; Adam's is dense.  The clip norm's own reads (the
    biases and the embedding rows; the matrices' sums come from the weight-gradient GEMMs) are left out."""
    V, H, L, T, B, p = CONFIGS[config]
    mats = L * (4 * H * H + 4 * H * H) + V * H
    img = L * (4 * H * H * 2 + 4 * H * H * 4) + V * H * 2
    small = L * 8 * H + V
    emb = V * H
    sgd = 12 * (mats + small) + 12 * min(T * B, V) * H + img
    adam = 28 * (mats + small + emb) + img
    return sgd, adam


def _torch_arm(config, xs, ys, warmup, steps, rounds):
    from oracle import torch_port as P
    V, H, L, T, B, p = CONFIGS[config]
    torch.manual_seed(0)
    model = P.TorchLstmLm(V, H, L, p, 0.04).cuda()
    model.train()
    opt = torch.optim.Adam(model.parameters(), lr=0.0, fused=True)
    states = [model.zero_state(B)]

    def run(n):
        s = torch.cuda.current_stream()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        for i in range(n):
            opt.zero_grad(set_to_none=True)
            st = [(h.detach(), c.detach()) for h, c in states[0]]
            logits, st = model(xs[i % WINDOWS], st)
            P.softmax_nll_times_batch(logits, ys[i % WINDOWS]).backward()
            torch.nn.utils.clip_grad_norm_(model.parameters(), 0.25)
            opt.step()
            states[0] = st
        b.record(s)
        b.synchronize()
        return a.elapsed_time(b) / n
    run(warmup)
    return [run(steps) for _ in range(rounds)]


def bench(config, warmup, steps, rounds):
    xs, ys = _data(config)
    rows = []
    for lazy in (False, True):
        trs = _trainers(config, lazy, xs, ys, warmup)
        ms = {"sgd": [], "adam": []}
        for _ in range(rounds):
            for opt in ("sgd", "adam"):
                ms[opt].append(window(trs[opt], xs, ys, steps, lr=0.0))
        row = dict(config=config, schedule="lazy" if lazy else "strict", ms_per_step_sgd=ms["sgd"],
                   ms_per_step_adam=ms["adam"])
        if not lazy:
            sgd_b, adam_b = update_bytes(config)
            sgd_ms, adam_ms = _update_ms(trs["sgd"], xs, ys), _update_ms(trs["adam"], xs, ys)
            row.update(update_ms_sgd=sgd_ms, update_ms_adam=adam_ms, update_bytes_sgd=sgd_b, update_bytes_adam=adam_b,
                       update_GBps_sgd=sgd_b / sgd_ms / 1e6, update_GBps_adam=adam_b / adam_ms / 1e6)
        rows.append(row)
        for t in trs.values():
            t.close()
    rows.append(dict(config=config, schedule="torch", ms_per_step_torch_adam=_torch_arm(config, xs, ys, warmup, steps,
                                                                                         rounds)))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--configs", default="small,medium,large")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_adam.py measures on a CUDA device; none is available")
    name, power = card()
    print(f"device: {name}, power limit {power}")
    out = dict(device=name, power_limit=power, warmup=args.warmup, steps=args.steps, results=[])
    for config in args.configs.split(","):
        for r in bench(config, args.warmup, args.steps, args.rounds):
            out["results"].append(r)
            if r["schedule"] == "torch":
                print(f"{config:6s} torch  cuDNN + Adam(fused) {' '.join(f'{v:.4f}' for v in r['ms_per_step_torch_adam'])}"
                      " ms/step", flush=True)
                continue
            s, a = min(r["ms_per_step_sgd"]), min(r["ms_per_step_adam"])
            line = (f"{config:6s} {r['schedule']:6s} sgd {' '.join(f'{v:.4f}' for v in r['ms_per_step_sgd'])} | "
                    f"adam {' '.join(f'{v:.4f}' for v in r['ms_per_step_adam'])} ms/step | best adam/sgd {a / s:.4f}")
            if "update_ms_adam" in r:
                line += (f" | update class sgd {r['update_ms_sgd']:.4f} ms ({r['update_GBps_sgd']:.0f} GB/s of "
                         f"{r['update_bytes_sgd'] / 1e9:.3f} GB), adam {r['update_ms_adam']:.4f} ms "
                         f"({r['update_GBps_adam']:.0f} GB/s of {r['update_bytes_adam'] / 1e9:.3f} GB)")
            print(line, flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
