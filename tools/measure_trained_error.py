#!/usr/bin/env python
"""Errors of both engines against the fp64 oracle at TRAINED weights (DESIGN.md section 5), over independent trainings.

Each run r trains the Medium recipe for one epoch of the Penn Treebank ids from torch seed r with the fused Trainer
(tensor-core engine, lazy update; the training is not bit-reproducible: the embedding-gradient scatter adds with fp32
atomics), then measures at a valid window with carried states what tests/test_gpu_trained_regime.py asserts -- the
regime statistics, eval forward, train- and eval-mode gradients, each layer alone at T = 35 and 140 (also against the
rounded-operand oracle), zrb_softmax_nll, zrb_sample -- and the Small training-trajectory parity of the two engines
from seed r.  Run 0 is the test's own fixture.  Prints one JSON line per run as it finishes (also appended to --out),
then the max and min of every number over the runs and the GPU's name and power limit.

    python tools/measure_trained_error.py [--runs 12] [--trajectory-steps 500] [--out runs.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from tests import _trained_regime as R  # noqa: E402


def gpu():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def flatten(d, pre=""):
    """Nested results -> {path: float}: (max-abs, l2) pairs and (worst row, rows) pairs get a suffix each."""
    out = {}
    for k, v in d.items():
        key = f"{pre}{k}"
        if isinstance(v, dict):
            out.update(flatten(v, key + "/"))
        elif isinstance(v, tuple) and isinstance(v[1], int):
            out[key + " worst_row"] = float(v[0])
        elif isinstance(v, tuple):
            out[key + " max_abs"], out[key + " l2"] = float(v[0]), float(v[1])
        else:
            out[key] = float(v)
    return out


def one_run(seed, trajectory_steps):
    t = R.train(R.MEDIUM, seed=seed)
    pt = R.Point(t["params"])
    out = {"train": {k: t[k] for k in ("seconds", "ppl_init", "ppl")}, "regime": pt.regime()}
    for e in ("tc", "simt"):
        out[e] = {"eval_forward": R.eval_forward(pt, e)}
        out[e]["train_loss"], out[e]["train_grads"] = R.train_grads(pt, e)
        out[e]["eval_grads"] = R.eval_grads(pt, e)
    out["layer_unit"] = {f"T={T}": R.layer_unit(pt, T) for T in (pt.c["T"], R.LONG_T)}
    out["softmax_nll"] = {f"V={V}": R.softmax_nll(pt, V) for V in (10000, 9999)}
    out["sampler"] = R.sampler(pt)
    out["trajectory_small"] = R.trajectory(trajectory_steps, seed=seed)
    return flatten(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=12)
    ap.add_argument("--trajectory-steps", type=int, default=500)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    runs = []
    for seed in range(args.runs):
        r = one_run(seed, args.trajectory_steps)
        runs.append(r)
        line = json.dumps({"seed": seed, **r})
        print(line, flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(line + "\n")
    keys = sorted(runs[0])
    print(json.dumps({"gpu": gpu(), "runs": len(runs),
                      "max": {k: max(r[k] for r in runs) for k in keys},
                      "min": {k: min(r[k] for r in runs) for k in keys}}, indent=1))


if __name__ == "__main__":
    main()
