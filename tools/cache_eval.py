#!/usr/bin/env python
"""Neural-cache evaluation of a trained checkpoint (Grave, Joulin & Usunier 2017; DESIGN.md section 12).

    python tools/train_ptb.py --recipe medium --seed 0 --save ckpt.pt
    python tools/cache_eval.py ckpt.pt --size 100,500,2000 --eval_batch_size 20 --json out/cache_medium.json

For every cache size W, theta is tuned on a grid over the validation set (one pass per theta, keeping p_model and
p_cache of every token) and lambda on the host from the same per-token probabilities, as the paper does.  Validation and
test perplexity with the tuned (theta, lambda) are reported next to the no-cache perplexity of the same checkpoint; the
test number is a device pass through Trainer.perplexity(cache=).
"""
import argparse, json, math, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch

ap = argparse.ArgumentParser()
ap.add_argument("checkpoint", help="a state_dict saved by tools/train_ptb.py --save")
ap.add_argument("--data", default=None, help="directory with ptb.{train,valid,test}.txt (default: the id fixture)")
ap.add_argument("--ids", default=os.path.join(ROOT, "tests", "golden", "ptb_ids.npz"))
ap.add_argument("--size", default="100,500,2000", help="cache sizes W, comma-separated")
ap.add_argument("--thetas", default="0,0.02,0.05,0.1,0.15,0.2,0.3,0.5,0.7,1.0")
ap.add_argument("--lambdas", default=",".join(f"{0.05 * i:.2f}" for i in range(20)))
ap.add_argument("--eval_batch_size", type=int, default=20)
ap.add_argument("--seq_length", type=int, default=35)
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
        return enc(vld), enc(tst)
    d = np.load(args.ids)
    return d["valid"].astype(np.int64).reshape(-1, 1), d["test"].astype(np.int64).reshape(-1, 1)


from generate import load_model                       # pytorch- and custom-layout checkpoints alike

dev = torch.device("cuda", 0)
model = load_model(args.checkpoint, args.engine)
V, H, L = model.embed.W.shape[0], model.hidden_size, model.layer_num
if model.lstm_type == "custom":
    # the Trainer drives the pytorch layout: the same weights with the custom cell's gate blocks permuted, which is
    # what the library computes with for a custom-layout model
    src = model
    model = zaremba_b200.Model(V, H, L, 0.0, 0.0, engine=args.engine)
    with torch.no_grad():
        for p, w in zip(model.ordered_parameters(), src._lib_weights()):
            p.copy_(w)
model = model.to(dev)
model.eval()
EB, T = args.eval_batch_size, args.seq_length
tr = zaremba_b200.Trainer(model, EB, T)
vld, tst = load_data()
vld_b = zaremba_b200.minibatch(vld, EB, T)
tst_b = zaremba_b200.minibatch(tst, EB, T)
thetas = [float(v) for v in args.thetas.split(",")]
lambdas = [float(v) for v in args.lambdas.split(",")]


def probs_pass(batches, cache, theta):
    """One pass with the cache: p_model and p_cache of every token (float64 on the host), in window order."""
    tr.reset_states()
    cache.reset()
    pm, pc = [], []
    for x, y in batches:
        _, p, c = tr.eval_step(x.to(dev).contiguous(), y.to(dev).contiguous(), want_probs=True, cache=cache,
                               theta=theta, lam=0.0)
        pm.append(p.double().clone()); pc.append(c.double().clone())
    return torch.cat(pm).cpu().numpy(), torch.cat(pc).cpu().numpy()


def host_ppl(pm, pc, lam):
    p = (1.0 - lam) * pm + lam * pc
    p[:EB] = pm[:EB]                    # every stream's first token: the cache is empty, p = p_model
    return math.exp(-np.log(p).mean())


base_v, base_t = tr.perplexity(vld_b), tr.perplexity(tst_b)
print(f"checkpoint {args.checkpoint}: V={V} H={H} L={L}, eval batch {EB}: no cache valid {base_v:.3f} test {base_t:.3f}")
out = {"checkpoint": os.path.basename(args.checkpoint), "hidden": H, "layers": L, "eval_batch_size": EB,
       "engine": args.engine, "no_cache": {"valid": base_v, "test": base_t}, "cache": [],
       "gpu": torch.cuda.get_device_name(0)}
for W in [int(v) for v in args.size.split(",")]:
    cache = zaremba_b200.NeuralCache(model.layer_sizes[-1], EB, W, T)   # keys: the last layer's output
    best = (float("inf"), 0.0, 0.0)
    for theta in thetas:
        pm, pc = probs_pass(vld_b, cache, theta)
        for lam in lambdas:
            best = min(best, (host_ppl(pm, pc, lam), theta, lam))
    ppl_v, theta, lam = best
    dev_v = tr.perplexity(vld_b, cache=cache, theta=theta, lam=lam)
    ppl_t = tr.perplexity(tst_b, cache=cache, theta=theta, lam=lam)
    print(f"W={W}: theta {theta} lambda {lam}: valid {ppl_v:.3f} (device pass {dev_v:.3f}) test {ppl_t:.3f} "
          f"(no cache {base_t:.3f})", flush=True)
    out["cache"].append({"size": W, "theta": theta, "lambda": lam, "valid": ppl_v, "valid_device": dev_v, "test": ppl_t})
    cache.close()
print(json.dumps(out))
if args.json:
    os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
    json.dump(out, open(args.json, "w"), indent=1)
