#!/usr/bin/env python
"""Sample text from a trained model with `Model.generate` (zrb_generate: prefill and decode loop on the device).

    python tools/train_ptb.py --recipe medium --save medium.pt
    python tools/generate.py medium.pt --data DIR --prompt "the company said" -n 30 --top_p 0.9
    python tools/generate.py medium.pt --prompt_ids 12,7,401 --batch 4 --temperature 0.8 --top_k 40
    python tools/generate.py --shape large --batch 20 --time     # decode speed with random weights at a BASELINE shape
    python tools/generate.py medium.pt --data DIR --prompt "the company" -n 20 --beams 8 --eos 0   # beam search
    python tools/generate.py --shape large --batch 4 --beams 8 --time

The checkpoint is a state_dict with the reference's key names (`train_ptb.py --save`); the model's shape and layout
are read from it.  `--data` names the directory of ptb.train.txt: words are then mapped with the reference's
vocabulary rule (tools/ptb_vocab.py, shared with train_ptb.py) and samples print as words, else as ids.

--time reports the decode loop after warm-up, timed with CUDA events: ms per decode step (one T = 1 forward and one
sampler launch per token) end to end and as device time alone, tokens/s over the B rows (end to end), and the bytes/s
the device time achieves against the bytes a decode step must read -- the fp16 weight images the forward streams
(input and recurrent matrices of every layer, the projection), computed from the shapes -- together with the
device's name and power limit.  It also times the sampler alone on a [B,V] score matrix (device time), to state its
share of a step.

--beams K runs `Model.beam_search` instead: the K most likely continuations of each prompt with their summed
log-probabilities (`--eos ID` freezes a hypothesis at that token; in the PTB vocabulary '<eos>', the newline, is id 0).
With --time the decode step covers one T = 1 forward of the B*K rows and the two beam kernels (top-K selection per
row; merge per prompt with the state reorder), whose device time per step is taken from a torch.profiler trace of one
search call.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

SHAPES = {"small": 200, "medium": 650, "large": 1500}   # hidden sizes of the README recipes; V = 10000, L = 2


def load_model(path, engine):
    import zaremba_b200
    sd = torch.load(path, map_location="cpu")
    if not any(k.endswith(".W_x") for k in sd):   # pytorch layout: V, E and the layer widths from the shapes
        return zaremba_b200.model_from_state_dict(sd, tied=False, engine=engine)
    V, H = sd["embed.W"].shape
    L = sum(1 for k in sd if k.endswith(".W_x"))
    m = zaremba_b200.Model(V, H, L, 0.0, 0.0, "custom", engine=engine)
    m.load_state_dict(sd)
    return m


def weight_image_bytes(model):
    """fp16 bytes a decode step reads from the weight images: per layer W_ih [4H_l, pad(In_l)] and W_hh [4H_l, pad(H_l)],
    and fc.W [V, pad(H_{L-1})] (pad: to 64 columns); fp32 biases besides."""
    pad = lambda n: (n + 63) // 64 * 64
    ins = [model.embed_size, *model.layer_sizes[:-1]]
    V, nb = model.vocab_size, 0
    for In, H in zip(ins, model.layer_sizes):
        nb += 2 * 4 * H * (pad(In) + pad(H)) + 4 * 2 * 4 * H
    return nb + 2 * V * pad(model.layer_sizes[-1]) + 4 * V


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or "unknown"
    except Exception:
        return "unknown"


def event_ms(fn, reps, hold=False):
    """Milliseconds per call between CUDA events.  hold: a spin kernel first keeps the stream busy while the host
    enqueues all calls, so they run back to back and the interval is device time alone (no host gaps)."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if hold:
        torch.cuda._sleep(int(2e8))                           # ~0.1 s at 1.98 GHz
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("checkpoint", nargs="?", help="state_dict saved by tools/train_ptb.py --save")
    ap.add_argument("--shape", choices=sorted(SHAPES), help="random weights at this shape instead of a checkpoint")
    ap.add_argument("--data", help="directory with ptb.train.txt: prompts and samples as words")
    ap.add_argument("--prompt", default=None, help="prompt words (needs --data)")
    ap.add_argument("--prompt_ids", default=None, help="comma-separated prompt token ids")
    ap.add_argument("-n", "--n_new", type=int, default=30)
    ap.add_argument("--batch", type=int, default=1, help="samples drawn side by side from the same prompt")
    ap.add_argument("--temperature", type=float, default=1.0)
    ap.add_argument("--top_k", type=int, default=0)
    ap.add_argument("--top_p", type=float, default=1.0)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--beams", type=int, default=0, help="beam search with this many beams instead of sampling")
    ap.add_argument("--eos", type=int, default=None, help="--beams: token id that ends a hypothesis")
    ap.add_argument("--engine", choices=["tc", "simt"], default="tc")
    ap.add_argument("--time", action="store_true", help="time the decode loop (CUDA events, after warm-up)")
    ap.add_argument("--steps", type=int, default=400, help="decode steps per timed call (--time)")
    ap.add_argument("--json", default=None, help="write the --time figures here")
    args = ap.parse_args()
    if bool(args.checkpoint) == bool(args.shape):
        ap.error("give a checkpoint or --shape")
    dev = torch.device("cuda", torch.cuda.current_device())
    if args.checkpoint:
        model = load_model(args.checkpoint, args.engine)
    else:
        import zaremba_b200
        torch.manual_seed(args.seed)
        model = zaremba_b200.Model(10000, SHAPES[args.shape], 2, 0.0, 0.05, engine=args.engine)
    model = model.to(dev).eval()
    V, H, L, B = model.vocab_size, model.hidden_size, model.layer_num, args.batch

    words = w2i = None
    if args.data:
        from ptb_vocab import read_words, vocabulary
        words, w2i = vocabulary(read_words(args.data, "ptb.train.txt"))
        if len(words) != V:
            raise SystemExit(f"the vocabulary of {args.data} has {len(words)} words, the model {V}")
    if args.prompt is not None:
        if w2i is None:
            raise SystemExit("--prompt takes words and needs --data; use --prompt_ids for ids")
        unknown = [w for w in args.prompt.split() if w not in w2i]
        if unknown:
            raise SystemExit(f"not in the vocabulary: {unknown}")
        ids = [w2i[w] for w in args.prompt.split()]
    elif args.prompt_ids is not None:
        ids = [int(t) for t in args.prompt_ids.split(",")]
    else:
        ids = [w2i["<eos>"] if w2i and "<eos>" in w2i else 0]
    prompt = torch.tensor(ids, dtype=torch.int64).view(-1, 1).expand(-1, B).contiguous()
    kw = dict(temperature=args.temperature, top_k=args.top_k, top_p=args.top_p, seed=args.seed)
    show = (lambda t: " ".join(words[i] for i in t)) if words else (lambda t: " ".join(map(str, t)))
    if args.beams:
        return beams(model, prompt, ids, args, show)

    tokens, logprobs, _ = model.generate(prompt, args.n_new, **kw)
    for b in range(B):
        col = tokens[:, b].tolist()
        print(f"[{b}] {show(ids)} | {show(col)}   (mean log-prob {logprobs[:, b].mean().item():.3f})")

    if not args.time:
        return
    from zaremba_b200 import sample
    n = args.steps
    one = prompt[-1:]
    for _ in range(3):                                        # warm-up: modules, weight images, plans
        model.generate(one, n, **kw)
    step_ms = event_ms(lambda: model.generate(one, n, **kw), 5) / n
    device_step_ms = event_ms(lambda: model.generate(one, n, **kw), 1, hold=True) / n
    scores = torch.randn(B, V, device=dev) * 2
    sample(scores, pos=1, **kw)
    sample_ms = event_ms(lambda: sample(scores, pos=1, **kw), 200, hold=True)
    nbytes = weight_image_bytes(model)
    out = {"device": torch.cuda.get_device_name(dev), "power_limit": power_limit(), "engine": args.engine,
           "V": V, "H": H, "L": L, "B": B, "decode_steps": n, "ms_per_step": round(step_ms, 4),
           "device_ms_per_step": round(device_step_ms, 4),
           "tokens_per_s": round(B * 1e3 / step_ms, 1), "weight_image_bytes": nbytes,
           "achieved_GB_per_s": round(nbytes / (device_step_ms * 1e-3) / 1e9, 1), "sampler_ms": round(sample_ms, 4),
           "sampler_share": round(sample_ms / device_step_ms, 4),
           "sampling": {k: v for k, v in kw.items() if k != "seed"}}
    print(json.dumps(out))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


def beam_kernel_ms(model, prompt, n, K, eos):
    """Device ms per decode step of the two beam kernels, from a torch.profiler trace of one search call."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model.beam_search(prompt, n, K, eos=eos)
        torch.cuda.synchronize()
    us = {"row": 0.0, "merge": 0.0}
    for e in prof.events():
        for k in us:
            if e.device_type == DeviceType.CUDA and f"beam_{k}_kernel" in e.name:
                us[k] += e.time_range.elapsed_us()
    return {k: v / 1e3 / n for k, v in us.items()}


def beams(model, prompt, ids, args, show):
    B, K = prompt.shape[1], args.beams
    model._context(min(prompt.shape[0], 64), B * K)
    tokens, logprobs, scores, _ = model.beam_search(prompt, args.n_new, K, eos=args.eos)
    for b in range(B):
        for k in range(K):
            print(f"[{b}.{k}] {show(ids)} | {show(tokens[:, b, k].tolist())}   (score {scores[b, k].item():.3f})")
    if not args.time:
        return
    n = args.steps
    one = prompt[-1:]
    for _ in range(3):                                        # warm-up: modules, weight images, plans, scratch
        model.beam_search(one, n, K, eos=args.eos)
    step_ms = event_ms(lambda: model.beam_search(one, n, K, eos=args.eos), 5) / n
    device_step_ms = event_ms(lambda: model.beam_search(one, n, K, eos=args.eos), 1, hold=True) / n
    kern = beam_kernel_ms(model, one, n, K, args.eos)
    from zaremba_b200 import _lib
    V, H, L = model.vocab_size, model.hidden_size, model.layer_num
    out = {"device": torch.cuda.get_device_name(), "power_limit": power_limit(), "engine": args.engine,
           "V": V, "H": H, "L": L, "B": B, "beams": K, "rows": B * K, "eos": args.eos, "decode_steps": n,
           "persistent": bool(args.engine == "tc" and _lib.rec_plans(model._ctx)["fwd"]["ok"]),
           "ms_per_step": round(step_ms, 4), "device_ms_per_step": round(device_step_ms, 4),
           "beam_row_ms": round(kern["row"], 4), "beam_merge_ms": round(kern["merge"], 4),
           "beam_share": round((kern["row"] + kern["merge"]) / device_step_ms, 4),
           "step_bytes": weight_image_bytes(model) + B * K * V * 4}
    print(json.dumps(out))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
