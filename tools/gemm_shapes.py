"""Time every GEMM of the Small / Medium / Large train steps at its exact shape, on both epilogues.

    python tools/gemm_shapes.py --out <dir> [--reps 200] [--configs small,medium,large]

Per call and per side (the default epilogue, and ZRB_GEMM_EPI=direct -- read at every launch, so both run in this
process, alternating): ms per call from CUDA events over --reps launches after warm-up, algorithmic TFLOP/s
(2*M*N*K / time), work items and rounds of the persistent grid.  The modes zrb_gemm_f16 does not reach (bias2, the
dual weight-gradient launch with sum-of-squares slots, the programmatic-dependent launches) are timed inside one fused
Large train step with torch.profiler (CUDA activities, a run of its own per side): kernel name -> total us.  Writes
gemm_shapes.json (with the GPU name, power limit and SM clock read in the same run) and the profiler tables to --out.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

GBM, GBK = 128, 64
CONFIGS = {"small": (200, 20, 20), "medium": (650, 35, 20), "large": (1500, 35, 20)}
V = 10000


def cdiv(a, b):
    return (a + b - 1) // b


def plan(M, N, K, can_split, nsm, sumsq, direct):
    """gemm_tc.cu choose_tiles and the pair plan restated: (tile width, splits, work items, rounds, tile rows)."""
    kb = cdiv(K, GBK)
    tm = cdiv(M, GBM)
    t256 = tm * cdiv(N, 256)
    if can_split and t256 * 2 <= nsm and t256 * 2 >= (nsm * 4) // 10 and kb // 2 >= 8:
        bn, sp = 256, 2
    else:
        bn = 256 if t256 >= (nsm * 9) // 10 else 128
        t128 = tm * cdiv(N, 128)
        if not direct and not sumsq and bn == 256 and cdiv(t256, nsm) * 2 > cdiv(t128, nsm) and t128 * 2 > nsm:
            bn = 128
        sp = 2 if (can_split and tm * cdiv(N, bn) * 2 <= nsm and kb >= 8) else 1
    items = tm * cdiv(N, bn) * sp
    tm64 = cdiv(M, 64)
    if sp == 2 and bn == 256 and not direct and tm64 > tm:
        # the pair plan (gemm_f16_tc_pair_kernel): 64-row items, two per 2-CTA cluster, taken when all its clusters are
        # resident at once (assumed here: nsm / 2 of them, as on a 132-SM H100); items = CTAs, a copy included
        tn = cdiv(N, bn)
        pairs = 2 * ((tm64 // 2) * tn + ((tn + 1) // 2 if tm64 % 2 else 0))
        if pairs <= nsm // 2:
            return bn, sp, 2 * pairs, 2 * pairs / nsm, 64
    return bn, sp, items, items / nsm, GBM


def calls(cfg):
    H, T, B = CONFIGS[cfg]
    Nt = T * B
    # (class, what, M, N, K, a_mn, b_mn, bias, layers per step)
    return [("gemm_in", "X*W_ih^T (+b_ih+b_hh)", Nt, 4 * H, H, 0, 0, True, 2),
            ("proj_fwd", "A*W_fc^T + b_fc", Nt, V, H, 0, 0, True, 1),
            ("proj_bwd", "dS*W_fc", Nt, H, V, 0, 1, False, 1),
            ("gemm_dx", "dG*W_ih", Nt, H, 4 * H, 0, 1, False, 2),
            ("gemm_wgrad", "dS^T*A (dW_fc)", V, H, Nt, 1, 1, False, 1),
            ("gemm_wgrad", "dG^T*X (dW_ih; dW_hh same shape)", 4 * H, H, Nt, 1, 1, False, 4)]


def set_side(side):
    os.environ.pop("ZRB_GEMM_EPI", None)
    if side == "direct":
        os.environ["ZRB_GEMM_EPI"] = "direct"


def time_call(lib, _lib, M, N, K, a_mn, b_mn, use_bias, reps, sides):
    def op(rows, k, mn):
        inner, outer = (rows, k) if mn else (k, rows)
        ld = cdiv(inner, 8) * 8
        return torch.randn(outer, ld, device="cuda").half(), ld
    A, lda = op(M, K, a_mn)
    Bm, ldb = op(N, K, b_mn)
    C = torch.empty(M, N, device="cuda")
    bias = torch.randn(N, device="cuda") if use_bias else None
    stream = torch.cuda.current_stream().cuda_stream

    def launch():
        _lib.check(lib.zrb_gemm_f16(_lib.ptr(A), lda, a_mn, _lib.ptr(Bm), ldb, b_mn, _lib.ptr(C), N, M, N, K, 1.0,
                                    _lib.ptr(bias), 0, stream))
    res = {s: [] for s in sides}
    for rnd in range(3):                      # alternate the sides three times, keep the best round of each
        for side in sides:
            set_side(side)
            for _ in range(10):
                launch()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                launch()
            e1.record()
            e1.synchronize()
            res[side].append(e0.elapsed_time(e1) / reps)
    set_side("new")
    return {s: min(v) for s, v in res.items()}


def profile_step(side, out_dir, steps=3):
    """One fused Large train step (lazy update, the bench's schedule) under torch.profiler: kernel -> total us."""
    import zaremba_b200
    set_side(side)
    H, T, B = CONFIGS["large"]
    torch.manual_seed(0)
    m = zaremba_b200.Model(V, H, 2, 0.65, 0.04).cuda()
    m.train()
    tr = zaremba_b200.Trainer(m, B, T, lazy_update=True)
    g = torch.Generator().manual_seed(1)
    data = torch.randint(0, V, (B, (steps + 4) * T + 1), generator=g).cuda()

    def step(i):
        x = data[:, i * T:(i + 1) * T].t().contiguous()
        y = data[:, i * T + 1:(i + 1) * T + 1].t().contiguous()
        tr.train_step(x, y, 1.0, 5.0)
    for i in range(3):
        step(i)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(steps):
            step(3 + i)
        tr.flush()
        torch.cuda.synchronize()
    table = {}
    for ev in prof.key_averages():
        if ev.device_type.name == "CUDA" or getattr(ev, "self_device_time_total", 0) > 0:
            us = getattr(ev, "self_device_time_total", None)
            if us is None:
                us = ev.self_cuda_time_total
            if us > 0:
                table[ev.key] = round(us / steps, 2)
    with open(os.path.join(out_dir, f"profile_large_{side}.txt"), "w") as f:
        for k, v in sorted(table.items(), key=lambda kv: -kv[1]):
            f.write(f"{v:10.1f} us/step  {k}\n")
    tr.close()
    del tr, m
    set_side("new")
    return table


def gpu_info():
    q = ["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"]
    try:
        line = subprocess.run(q, capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, sm, smax = [s.strip() for s in line.split(",")]
        return dict(name=name, power_limit=power, sm_clock=sm, sm_clock_max=smax)
    except Exception as e:                     # noqa: BLE001 -- the numbers still stand with the torch name
        return dict(name=torch.cuda.get_device_name(0), error=str(e))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--configs", default="small,medium,large")
    ap.add_argument("--no-profile", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("gemm_shapes.py needs a GPU")
    os.makedirs(a.out, exist_ok=True)
    from zaremba_b200 import _lib
    lib = _lib.load()
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    info = gpu_info()
    print(f"# {info} | {nsm} SMs")
    sides = ["direct", "new"]
    rows = []
    for cfg in a.configs.split(","):
        for cls, what, M, N, K, a_mn, b_mn, bias, per_step in calls(cfg):
            t = time_call(lib, _lib, M, N, K, a_mn, b_mn, bias, a.reps, sides)
            flop = 2.0 * M * N * K
            for side in sides:
                bn, sp, items, rounds, bm = plan(M, N, K, True, nsm, False, side == "direct")
                r = dict(config=cfg, cls=cls, what=what, M=M, N=N, K=K, side=side, ms=t[side],
                         tflops=flop / t[side] / 1e9, tile_m=bm, tile_n=bn, splits=sp, work_items=items, rounds=rounds,
                         calls_per_step=per_step)
                rows.append(r)
                print(f"{cfg:6s} {cls:10s} {M:5d}x{N:5d}x{K:5d} {side:6s} {t[side]*1e3:8.1f} us "
                      f"{r['tflops']:6.1f} TFLOP/s  {bm}x{bn} x{sp}: {items} items, {rounds:.2f} rounds  ({what})")
    prof = {}
    if not a.no_profile:
        for side in sides:
            prof[side] = profile_step(side, a.out)
            gemm = sum(v for k, v in prof[side].items() if "gemm_f16_tc_kernel" in k or "gemm_f16_tc_pair_kernel" in k)
            total = sum(prof[side].values())
            print(f"# profile Large step, {side}: GEMM kernels {gemm:.1f} us of {total:.1f} us kernel time per step")
            for k, v in sorted(prof[side].items(), key=lambda kv: -kv[1])[:12]:
                print(f"#   {v:8.1f} us  {k[:110]}")
    with open(os.path.join(a.out, "gemm_shapes.json"), "w") as f:
        json.dump(dict(gpu=info, num_sms=nsm, reps=a.reps, calls=rows, profile_us_per_step=prof), f, indent=1)


if __name__ == "__main__":
    main()
