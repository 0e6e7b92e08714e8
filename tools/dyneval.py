#!/usr/bin/env python
"""Dynamic evaluation of a trained checkpoint (Krause, Kahembwe, Murray & Renals 2018; DESIGN.md section 14).

    python tools/train_ptb.py --recipe medium --seed 0 --save ckpt.pt
    python tools/dyneval.py ckpt.pt --eval_batch_size 1,20 --json out/dyneval_medium.json

A checkpoint whose embed.W equals fc.W (`train_ptb.py --tied`) is adapted as a tied model: E counts once.  The RMS
rule's statistics come from training windows (`--stats_windows`, default all) at theta_g, on a Trainer of their own
shape.  For each rule (RMS
with the global prior, SGD) and each eval batch, lr is tuned on a grid over the validation set with lambda = 0, then
lambda on a grid at that lr; validation and test perplexity with the tuned pair are reported next to the static
perplexity of the same checkpoint.  Every pass starts from the checkpoint's weights (Trainer.dynamic_perplexity restores
them).
"""
import argparse, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch

ap = argparse.ArgumentParser()
ap.add_argument("checkpoint", help="a state_dict saved by tools/train_ptb.py --save")
ap.add_argument("--data", default=None, help="directory with ptb.{train,valid,test}.txt (default: the id fixture)")
ap.add_argument("--ids", default=os.path.join(ROOT, "tests", "golden", "ptb_ids.npz"))
ap.add_argument("--eval_batch_size", default="1,20", help="comma-separated")
ap.add_argument("--seq_length", type=int, default=None, help="evaluation window (default: 5 for B = 1, else 35)")
ap.add_argument("--stats_batch_size", type=int, default=20)
ap.add_argument("--stats_seq_length", type=int, default=35)
ap.add_argument("--stats_windows", type=int, default=0, help="training windows for the statistics (0: all)")
ap.add_argument("--rms_lrs", default="1e-5,3e-5,1e-4,3e-4,1e-3")
ap.add_argument("--sgd_lrs", default="0.003,0.01,0.03,0.1,0.3")
ap.add_argument("--lambdas", default="0.001,0.003,0.01,0.03")
ap.add_argument("--eps", type=float, default=2e-5)
ap.add_argument("--engine", default="tc", choices=["tc", "simt"])
ap.add_argument("--json", default=None)
args = ap.parse_args()

import zaremba_b200


def load_data():
    if args.data:
        from ptb_vocab import read_words, vocabulary
        trn, vld, tst = (read_words(args.data, f"ptb.{s}.txt") for s in ("train", "valid", "test"))
        _, w2i = vocabulary(trn)
        enc = lambda toks: np.array([w2i[w] for w in toks]).reshape(-1, 1)
        return enc(trn), enc(vld), enc(tst)
    d = np.load(args.ids)
    return tuple(d[s].astype(np.int64).reshape(-1, 1) for s in ("train", "valid", "test"))


from generate import load_model                       # pytorch- and custom-layout checkpoints alike

dev = torch.device("cuda", 0)
src = load_model(args.checkpoint, args.engine)
V, H, L = src.embed.W.shape[0], src.hidden_size, src.layer_num
# a `train_ptb.py --tied` checkpoint carries E under both keys: adapt it as one matrix, as DESIGN section 14 counts it
tied = bool(torch.equal(src.embed.W, src.fc.W))


def fresh_model():
    """The checkpoint as a pytorch-layout model (the Trainer drives that layout; a custom-layout checkpoint's gate
    blocks are permuted as the library permutes them), tied when its embed.W and fc.W are equal."""
    m = zaremba_b200.Model(V, H, L, 0.0, 0.0, engine=args.engine, tied=tied)
    ws = src._lib_weights()
    if tied:
        ws = ws[:-2] + ws[-1:]          # E once: drop fc.W, keep fc.b
    with torch.no_grad():
        for p, w in zip(m.ordered_parameters(), ws, strict=True):
            p.copy_(w)
    m = m.to(dev)
    m.eval()
    return m


trn, vld, tst = load_data()
stats_b = zaremba_b200.minibatch(trn, args.stats_batch_size, args.stats_seq_length)
if args.stats_windows:
    stats_b = stats_b[:args.stats_windows]
out = {"checkpoint": os.path.basename(args.checkpoint), "hidden": H, "layers": L, "tied": tied, "engine": args.engine,
       "stats": {"windows": len(stats_b), "batch_size": args.stats_batch_size, "seq_length": args.stats_seq_length},
       "eps": args.eps, "gpu": torch.cuda.get_device_name(0), "runs": []}
# the statistics on a Trainer of their own shape, so that every evaluation Trainer keeps the recurrence plans of its
# own batch; the flat layout, and so the GradStats, is the same for every Trainer of this model configuration
t0 = time.time()
st_tr = zaremba_b200.Trainer(fresh_model(), args.stats_batch_size, args.stats_seq_length, data_parallel=False)
stats = st_tr.gradient_stats(stats_b)
print(f"statistics over {len(stats_b)} windows: r-bar {float(stats.mean):.4e} ({time.time() - t0:.1f} s)", flush=True)
out["stats"]["rms_mean"] = float(stats.mean)
del st_tr
for EB in [int(b) for b in args.eval_batch_size.split(",")]:
    T = args.seq_length or (5 if EB == 1 else 35)
    tr = zaremba_b200.Trainer(fresh_model(), EB, T, data_parallel=False)
    vld_b = zaremba_b200.minibatch(vld, EB, T)
    tst_b = zaremba_b200.minibatch(tst, EB, T)
    base_v, base_t = tr.perplexity(vld_b), tr.perplexity(tst_b)
    run = {"eval_batch_size": EB, "seq_length": T, "static": {"valid": base_v, "test": base_t}, "rules": {}}
    print(f"B={EB} T={T}: static valid {base_v:.3f} test {base_t:.3f}", flush=True)
    for rule, lrs, st in (("rms", args.rms_lrs, stats), ("sgd", args.sgd_lrs, None)):
        t0 = time.time()
        grid = []
        for lr in [float(v) for v in lrs.split(",")]:
            grid.append((tr.dynamic_perplexity(vld_b, lr, 0.0, st, args.eps), lr, 0.0))
        _, lr, _ = min(grid)
        for lam in [float(v) for v in args.lambdas.split(",")]:
            grid.append((tr.dynamic_perplexity(vld_b, lr, lam, st, args.eps), lr, lam))
        ppl_v, lr, lam = min(grid)
        ppl_t = tr.dynamic_perplexity(tst_b, lr, lam, st, args.eps)
        run["rules"][rule] = {"lr": lr, "lambda": lam, "valid": ppl_v, "test": ppl_t,
                              "grid": [{"lr": g[1], "lambda": g[2], "valid": g[0]} for g in grid],
                              "seconds": time.time() - t0}
        print(f"  {rule}: lr {lr:g} lambda {lam:g}: valid {ppl_v:.3f} test {ppl_t:.3f} "
              f"(static {base_v:.3f} / {base_t:.3f}; {time.time() - t0:.0f} s)", flush=True)
    out["runs"].append(run)
    del tr
    torch.cuda.empty_cache()
print(json.dumps(out))
if args.json:
    os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
    json.dump(out, open(args.json, "w"), indent=1)
