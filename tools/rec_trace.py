#!/usr/bin/env python
"""Phase timeline of the persistent recurrence kernels (zrb_prof_rec_trace): mean clocks per phase."""
import os, sys, json, ctypes as C
os.environ["ZRB_REC_TRACE"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import zaremba_b200
from zaremba_b200 import _lib
from bench import CONFIGS

c = CONFIGS[sys.argv[1] if len(sys.argv) > 1 else "large"]
V, H, L, T, B = c["V"], c["H"], c["L"], c["T"], c["B"]
torch.manual_seed(1)
m = zaremba_b200.Model(V, H, L, c["p"], c["winit"]).cuda(); m.train()
tr = zaremba_b200.Trainer(m, B, T)
g = torch.Generator().manual_seed(2)
for i in range(6):
    d = torch.randint(0, V, (B, T + 1), generator=g)
    tr.train_step(d[:, :T].t().contiguous().cuda(), d[:, 1:].t().contiguous().cuda(), c["lr"], c["clip"])
E = 8 + T * 8
buf = (C.c_int64 * (2 * E))()
n = _lib.load().zrb_prof_rec_trace(tr.ctx, buf, 2 * E)
assert n == 2 * E, n
raw = np.array(buf[:], dtype=np.int64).reshape(2, E)
launch, a = raw[:, :8], raw[:, 8:].reshape(2, T, 8)
# the 8 clock64 stamps of a step (CTA 0), both kernels:
#   barrier_seen     loader: the grid barrier of the step has passed, the operand copies are issued
#   mma_start        MMA warpgroup: the first operand piece has landed, the wgmma chain starts
#   acc_out          MMA warpgroup: chain drained, accumulators staged or pushed to their owners, arrival on bar_mma
#   acc_seen         cell warps: bar_mma completed
#   partials_landed  cell warps: every partial sum of this CTA's rows is in its shared memory (the K-split / cluster
#                    exchange; right after acc_seen when there is none)
#   cells_done       cell warps: cell math done, the next step's operand image stored
#   pre_arrive       after the cell warps' named barrier
#   arrived          after the release-add on the grid-barrier counter
names = ["barrier_seen", "mma_start", "acc_out", "acc_seen", "partials_landed", "cells_done", "pre_arrive", "arrived"]
out = {}
for d, nm in enumerate(["fwd", "bwd"]):
    x = a[d][2:T - 1]                       # steady-state steps
    step = np.diff(a[d][1:, 0]).mean()
    rel = (x - x[:, :1]).mean(0)
    out[nm] = {"clk_per_step": float(step), "phase_offsets_clk": dict(zip(names, [float(v) for v in rel])),
               # the launch's first steps: step 0 has no barrier to wait for but starts with the weight-slice load
               "step_starts_clk_rel_to_step0": [int(v - a[d][0, 0]) for v in a[d][:5, 0]],
               "step0_phase_offsets_clk": dict(zip(names, [int(v - a[d][0, 0]) for v in a[d][0]])),
               "whole_window_clk": int(a[d][T - 1, 7] - a[d][0, 0]),
               # where a launch's time goes outside the T steps (last layer's launch of the last step)
               "launch": {"cta0_entry_to_first_stamp_clk": int(a[d][0, 0] - launch[d][0]),
                          "last_arrival_to_cta0_exit_clk": int(launch[d][1] - a[d][T - 1, 7]),
                          "cta0_lifetime_clk": int(launch[d][1] - launch[d][0]),
                          "cta0_lifetime_ns": int(launch[d][3] - launch[d][2]),
                          "grid_lifetime_ns": int(launch[d][5] + launch[d][4]),
                          "first_cta_entry_to_cta0_entry_ns": int(launch[d][2] + launch[d][4]),
                          "cta0_exit_to_last_cta_exit_ns": int(launch[d][5] - launch[d][3])}}
print(json.dumps(out, indent=1))
