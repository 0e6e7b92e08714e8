#!/usr/bin/env python
"""main.py's job (train + validate + test on Penn Treebank) driven through the fused `zaremba_b200.Trainer`,
or -- `--impl cudnn` -- through the reference's own `--lstm_type pytorch` sequence of torch calls on the GPU
(oracle/torch_port.py: cuDNN nn.LSTM, eager loss, clip_grad_norm_, per-parameter SGD), same seed, same data,
same schedule: the "matched valid perplexity" half of BASELINE.json's target.

    python tools/train_ptb.py --recipe large                       # README.md:26 on the committed id fixture
    python tools/train_ptb.py --recipe small --impl cudnn --json out/ptb_small_cudnn.json
    python tools/train_ptb.py --data /root/reference/data --hidden_size 650 ...   # from the text files
    torchrun --nproc-per-node 8 tools/train_ptb.py --recipe large  # data parallel, batch_size rows per GPU

Same flags, data handling (main.py:44-74), LR schedule (main.py:105-106) and log lines (main.py:118-132) as the
reference; the step itself is one library call instead of ~30 eager launches.  (To run the UNMODIFIED main.py on
the drop-in Model instead, see INTEGRATION.md section A.)  Token ids come from `tests/golden/ptb_ids.npz`
(minted from the reference's text by tests/golden/make_ptb_ids.py with the reference's vocabulary rule) unless
`--data` names a directory with the ptb.*.txt files.  `--impl cudnn` is baseline/test infrastructure: it is the
only mode that imports `oracle/`.
"""
import argparse, json, math, os, sys, time, timeit
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

RECIPES = {   # README.md:20-27
    "small": dict(hidden_size=200, dropout=0.0, winit=0.1, seq_length=20, total_epochs=13, factor_epoch=4, factor=2.0,
                  max_grad_norm=5.0),
    "medium": dict(hidden_size=650, dropout=0.5, winit=0.05, seq_length=35, total_epochs=39, factor_epoch=6,
                   factor=1.2, max_grad_norm=5.0),
    "large": dict(hidden_size=1500, dropout=0.65, winit=0.04, seq_length=35, total_epochs=55, factor_epoch=14,
                  factor=1.15, max_grad_norm=10.0),
}

ap = argparse.ArgumentParser()
ap.add_argument("--recipe", choices=sorted(RECIPES), default=None, help="one of the README's three single-model recipes")
ap.add_argument("--impl", choices=["ours", "cudnn"], default="ours")
ap.add_argument("--data", default=None, help="directory with ptb.{train,valid,test}.txt (default: the id fixture)")
ap.add_argument("--ids", default=os.path.join(ROOT, "tests", "golden", "ptb_ids.npz"))
ap.add_argument("--layer_num", type=int, default=2)
ap.add_argument("--hidden_size", type=int, default=650)
ap.add_argument("--embed_size", type=int, default=None,
                help="embedding width E (default: --hidden_size); with --tied it must equal the last layer's width")
ap.add_argument("--layer_sizes", type=lambda s: tuple(int(v) for v in s.split(",")), default=None,
                help="one width per layer, e.g. AWD-LSTM's 1150,1150,400; sets --hidden_size and --layer_num")
ap.add_argument("--experts", type=int, default=None,
                help="a Mixture-of-Softmaxes head of this many softmaxes (Yang et al. 2018; e.g. 15 with --embed_size 280 "
                     "--layer_sizes 960,960,620 --tied)")
ap.add_argument("--mos_dropout", type=float, default=0.0, help="latent dropout of the --experts head")
ap.add_argument("--zoneout_cell", type=float, default=0.0,
                help="zoneout of the cell state (Krueger et al. 2017; the paper's LSTM setting is 0.5)")
ap.add_argument("--zoneout_hidden", type=float, default=0.0,
                help="zoneout of the hidden state (Krueger et al. 2017; the paper's LSTM setting is 0.05)")
ap.add_argument("--dropout", type=float, default=0.5)
ap.add_argument("--winit", type=float, default=0.05)
ap.add_argument("--batch_size", type=int, default=20)
ap.add_argument("--seq_length", type=int, default=35)
ap.add_argument("--learning_rate", type=float, default=1)
ap.add_argument("--total_epochs", type=int, default=39)
ap.add_argument("--factor_epoch", type=int, default=6)
ap.add_argument("--factor", type=float, default=1.2)
ap.add_argument("--max_grad_norm", type=float, default=5)
ap.add_argument("--seed", type=int, default=0)
ap.add_argument("--variational", action="store_true",
                help="variational dropout (Gal & Ghahramani 2016): masks fixed over each window, recurrent dropout")
ap.add_argument("--recurrent_dropout", type=float, default=None,
                help="p of the recurrent masks with --variational (default: --dropout)")
ap.add_argument("--tied", action="store_true",
                help="tie the embedding and softmax weights (Press & Wolf 2017): fc.W is embed.W")
ap.add_argument("--weight_drop", type=float, default=0.0,
                help="weight-dropped LSTM (Merity et al. 2018): DropConnect with this p on the hidden-to-hidden matrices")
ap.add_argument("--embed_dropout", type=float, default=0.0,
                help="embedding dropout (Merity et al. 2018): whole word types dropped with this p in each train step")
ap.add_argument("--ar", type=float, default=0.0,
                help="AR (Merity et al. 2018): alpha of the penalty on the last layer's dropped output (AWD: 2)")
ap.add_argument("--tar", type=float, default=0.0,
                help="TAR (Merity et al. 2018): beta of the penalty on the last layer's step-to-step change (AWD: 1)")
ap.add_argument("--asgd", action="store_true",
                help="NT-ASGD (Merity et al. 2018): start averaging the weights once validation stops improving "
                     "(AWD-LSTM's non-monotone trigger); validate, test and save with the average from then on")
ap.add_argument("--nonmono", type=int, default=5,
                help="--asgd: trigger when more than this many validations exist and this one is worse than the best "
                     "of all but the last NONMONO")
ap.add_argument("--asgd_from", type=int, default=None,
                help="start averaging at the start of this epoch (1-based), whatever validation does")
ap.add_argument("--optimizer", choices=["sgd", "adam"], default="sgd",
                help="adam: torch.optim.Adam after the clip, in place of SGD (DESIGN.md section 21); --learning_rate is "
                     "its lr and the schedule divides it as it divides SGD's.  --impl cudnn runs torch.optim.Adam(fused=True)")
ap.add_argument("--beta1", type=float, default=0.9, help="--optimizer adam: beta1 (Melis et al. 2018 use 0)")
ap.add_argument("--beta2", type=float, default=0.999, help="--optimizer adam: beta2")
ap.add_argument("--adam_eps", type=float, default=1e-8, help="--optimizer adam: eps (Melis et al. 2018 use 1e-9)")
ap.add_argument("--lazy_update", action="store_true",
                help="Trainer(lazy_update=True): upper-layer / fc weight updates run beside the next step's forward")
ap.add_argument("--eval_batch_size", type=int, default=None,
                help="batch size of the validation / test sweeps (default: --batch_size, like main.py)")
ap.add_argument("--epochs", type=int, default=None, help="stop after this many epochs (schedule unchanged)")
ap.add_argument("--json", default=None, help="write per-epoch validation perplexities, test perplexity, timing here")
ap.add_argument("--save", default=None, help="save the trained state_dict (reference key names) here")
args = ap.parse_args()
if args.recipe:
    for k, v in RECIPES[args.recipe].items():
        setattr(args, k, v)
if args.layer_sizes is not None:
    args.hidden_size, args.layer_num = args.layer_sizes[0], len(args.layer_sizes)
if args.impl == "cudnn" and (args.embed_size is not None or args.layer_sizes is not None):
    raise SystemExit("--embed_size / --layer_sizes are modes of --impl ours")
if args.impl == "cudnn" and (args.experts is not None or args.mos_dropout):
    raise SystemExit("--experts / --mos_dropout are modes of --impl ours")
if args.mos_dropout and args.experts is None:
    raise SystemExit("--mos_dropout needs --experts")
if args.impl == "cudnn" and (args.zoneout_cell or args.zoneout_hidden):
    raise SystemExit("--zoneout_cell / --zoneout_hidden are modes of --impl ours")
if args.embed_size is not None or args.layer_sizes is not None:
    from zaremba_b200.model import _check_widths
    try:
        _E, _sizes = _check_widths(args.hidden_size, args.layer_num, args.embed_size, args.layer_sizes)
    except ValueError as e:
        raise SystemExit(f"--embed_size / --layer_sizes: {e}")
    if args.tied and _E != _sizes[-1] and args.experts is None:
        raise SystemExit(f"--tied needs --embed_size equal to the last layer's width ({_E} != {_sizes[-1]})")


def data_init_text(root):                              # main.py:44-59
    from ptb_vocab import read_words, vocabulary
    trn, vld, tst = (read_words(root, f"ptb.{s}.txt") for s in ("train", "valid", "test"))
    words, w2i = vocabulary(trn)
    enc = lambda toks: np.array([w2i[w] for w in toks]).reshape(-1, 1)
    return enc(trn), enc(vld), enc(tst), len(words)


def data_init_ids(path):
    d = np.load(path)
    col = lambda a: a.astype(np.int64).reshape(-1, 1)
    return col(d["train"]), col(d["valid"]), col(d["test"]), int(d["vocab_size"])


import zaremba_b200
from zaremba_b200 import parallel

rank, local, world = parallel.init_from_env("nccl")
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
trn, vld, tst, vocab = data_init_text(args.data) if args.data else data_init_ids(args.ids)
B, T = args.batch_size, args.seq_length
trn_b = zaremba_b200.minibatch(parallel.shard_rows(trn, B, rank, world), B, T)
EB = args.eval_batch_size or B
vld_b = zaremba_b200.minibatch(vld, EB, T)
tst_b = zaremba_b200.minibatch(tst, EB, T)
torch.manual_seed(args.seed)

if args.impl == "ours":
    model = zaremba_b200.Model(vocab, args.hidden_size, args.layer_num, args.dropout, args.winit,
                               variational=args.variational, recurrent_dropout=args.recurrent_dropout,
                               tied=args.tied, weight_drop=args.weight_drop, embed_dropout=args.embed_dropout,
                               embed_size=args.embed_size, layer_sizes=args.layer_sizes, experts=args.experts,
                               mos_dropout=args.mos_dropout, zoneout_cell=args.zoneout_cell,
                               zoneout_hidden=args.zoneout_hidden).to(dev)
    if args.optimizer == "adam" and (args.asgd or args.asgd_from is not None):
        raise SystemExit("--asgd / --asgd_from average SGD iterates: not with --optimizer adam")
    tr = zaremba_b200.Trainer(model, B, T, lazy_update=args.lazy_update, ar=args.ar, tar=args.tar,
                              optimizer=args.optimizer, betas=(args.beta1, args.beta2), eps=args.adam_eps)
    # the corpus is staged on the device once (SURVEY 8f#2): 3 x [n_batches, T, B] int64
    trn_x = torch.stack([x for x, _ in trn_b]).contiguous().to(dev)
    trn_y = torch.stack([y for _, y in trn_b]).contiguous().to(dev)

    def train_epoch(lr, log):
        tr.reset_states()
        model.train()
        every = max(1, len(trn_b) // 10)
        for i in range(len(trn_b)):
            loss, norm = tr.train_step(trn_x[i], trn_y[i], lr, args.max_grad_norm)
            if i % every == 0:
                log(i, loss.item(), norm.item())

    def perplexity(batches):
        model.eval()
        return tr.perplexity(batches)

    def state_dict():
        if tr.averaged_steps:
            return {k: v.cpu() for k, v in tr.average_state_dict().items()}
        tr.flush()
        return {k: v.detach().cpu() for k, v in model.state_dict().items()}

    def averaged_perplexity(batches):
        """perplexity with the averaged weights once averaging has run (AWD-LSTM validates and tests the average)"""
        if not tr.averaged_steps:
            return perplexity(batches)
        with tr.averaged_weights():
            return perplexity(batches)
else:
    if world > 1:
        raise SystemExit("--impl cudnn is the reference's single-device path")
    if args.variational:
        raise SystemExit("--variational is a mode of --impl ours")
    if args.tied:
        raise SystemExit("--tied is a mode of --impl ours (the reference's cudnn path keeps embed.W and fc.W apart)")
    if args.weight_drop:
        raise SystemExit("--weight_drop is a mode of --impl ours")
    if args.embed_dropout:
        raise SystemExit("--embed_dropout is a mode of --impl ours")
    if args.ar or args.tar:
        raise SystemExit("--ar / --tar are modes of --impl ours")
    if args.asgd or args.asgd_from is not None:
        raise SystemExit("--asgd / --asgd_from are modes of --impl ours")
    from oracle import torch_port as P
    model = P.TorchLstmLm(vocab, args.hidden_size, args.layer_num, args.dropout, args.winit).to(dev)
    trn_d = [(x.to(dev), y.to(dev)) for x, y in trn_b]
    adam = (torch.optim.Adam(model.parameters(), lr=args.learning_rate, betas=(args.beta1, args.beta2),
                             eps=args.adam_eps, fused=True) if args.optimizer == "adam" else None)

    def adam_step(x, y, states, lr):
        """main.py:109-117 with torch.optim.Adam in place of the SGD loop"""
        adam.zero_grad(set_to_none=True)
        states = [(h.detach(), c.detach()) for h, c in states]
        logits, states = model(x, states)
        loss = P.softmax_nll_times_batch(logits, y)
        loss.backward()
        norm = torch.nn.utils.clip_grad_norm_(model.parameters(), args.max_grad_norm)
        for g in adam.param_groups:
            g["lr"] = lr
        adam.step()
        return loss, norm, states

    def train_epoch(lr, log):
        model.train()
        states = model.zero_state(B)
        every = max(1, len(trn_b) // 10)
        for i, (x, y) in enumerate(trn_d):
            if adam is not None:
                loss, norm, states = adam_step(x, y, states, lr)
            else:
                loss, norm, states = P.train_step(model, x, y, states, lr, args.max_grad_norm)
            if i % every == 0:
                log(i, loss.item(), float(norm))

    def perplexity(batches):                           # main.py:86-95
        model.eval()
        with torch.no_grad():
            losses, states = [], model.zero_state(EB)
            for x, y in batches:
                logits, states = model(x.to(dev), states)
                losses.append(P.softmax_nll_times_batch(logits, y.to(dev)).item() / EB)
        return float(np.exp(np.mean(losses)))

    averaged_perplexity = perplexity

    def state_dict():
        return {k: v.detach().cpu() for k, v in model.reference_state_dict().items()}

lr, tic, words_seen = args.learning_rate, timeit.default_timer(), 0
val_curve, epoch_secs = [], []
asgd_epoch = None                                      # 1-based epoch at whose start averaging began
n_epochs = args.total_epochs if args.epochs is None else min(args.epochs, args.total_epochs)
for epoch in range(n_epochs):
    if epoch > args.factor_epoch:                      # main.py:105-106
        lr = lr / args.factor
    e_words = [0]
    if args.asgd_from is not None and asgd_epoch is None and epoch + 1 >= args.asgd_from:
        tr.start_averaging()
        asgd_epoch = epoch + 1
        if rank == 0:
            print(f"averaging the weights from epoch {asgd_epoch} on (--asgd_from)", flush=True)

    def log(i, loss, norm, epoch=epoch):
        if loss != loss:                               # NaN: the run is dead, do not burn the remaining epochs
            if rank == 0:
                print(f"NON-FINITE train loss at epoch {epoch + 1}, batch {i}: aborting (seed {args.seed})", flush=True)
                if args.json:
                    json.dump({"impl": args.impl, "recipe": args.recipe, "seed": args.seed, "diverged": True,
                               "epoch": epoch + 1, "batch": i, "valid_ppl_per_epoch": [round(v, 3) for v in val_curve]},
                              open(args.json, "w"), indent=1)
            sys.exit(3)
        if rank == 0:
            toc = timeit.default_timer()
            seen = words_seen + (i + 1) * T * B * world
            print("batch no = {:d} / {:d}, train loss = {:.3f}, wps = {:d}, dw.norm() = {:.3f}, lr = {:.3f}, "
                  "since beginning = {:d} mins, cuda memory = {:.3f} GBs".format(
                      i, len(trn_b), loss / B, round(seen / (toc - tic)), norm, lr, round((toc - tic) / 60),
                      torch.cuda.max_memory_allocated() / 1024 ** 3), flush=True)

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    train_epoch(lr, log)
    torch.cuda.synchronize()
    epoch_secs.append(time.perf_counter() - t0)
    words_seen += len(trn_b) * T * B * world
    val = averaged_perplexity(vld_b)
    # AWD-LSTM's non-monotone trigger: more than nonmono earlier validations, and this one worse than the best of all
    # but the last nonmono of them.  Every rank computes the same validation, so every rank starts together.
    if args.asgd and asgd_epoch is None and len(val_curve) > args.nonmono and val > min(val_curve[:-args.nonmono]):
        tr.start_averaging()
        asgd_epoch = epoch + 2
        if rank == 0:
            print(f"validation stopped improving: averaging the weights from epoch {asgd_epoch} on", flush=True)
    val_curve.append(val)
    if rank == 0:
        print("Epoch : {:d} || Validation set perplexity : {:.3f}".format(epoch + 1, val))
        print("*************************************************\n", flush=True)
tst_ppl = averaged_perplexity(tst_b)
if rank == 0:
    print("Test set perplexity : {:.3f}".format(tst_ppl))
    print("Training is over.")
    if args.json:
        steps = len(trn_b)
        out = {"impl": args.impl, "recipe": args.recipe, "args": {k: v for k, v in vars(args).items()
                                                                 if k not in ("json", "save", "data", "ids")},
               "world": world, "vocab": vocab, "steps_per_epoch": steps, "epochs_run": n_epochs,
               "valid_ppl_per_epoch": [round(v, 3) for v in val_curve], "test_ppl": round(tst_ppl, 3),
               "train_seconds_per_epoch_median": float(np.median(epoch_secs)),
               "train_tokens_per_s_median_epoch": steps * T * B * world / float(np.median(epoch_secs)),
               "total_wall_s": timeit.default_timer() - tic, "gpu": torch.cuda.get_device_name(0),
               "data": os.path.basename(args.data or args.ids),
               "asgd_start_epoch": asgd_epoch, "averaged_steps": tr.averaged_steps if args.impl == "ours" else 0}
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        json.dump(out, open(args.json, "w"), indent=1)
    if args.save:
        torch.save(state_dict(), args.save)
