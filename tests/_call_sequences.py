"""Seeded call sequences over the Trainer / Model entry points, for tests/test_gpu_call_sequences.py.

A sequence is a list of operations (name, args) drawn from ALPHABET by a generator that follows the documented rules:
no train step inside averaged_weights(), dynamic-evaluation windows no wider than the Trainer's batch, no
data-parallel calls.  Each refusal the rules imply is an operation of its own ("refuse").  The generator also keeps a
model of the state the GPU test is about -- whether lazy weight updates are pending, whether averaging is on, whether
the average is swapped in, the weight-drop p, the context's window length -- and records it beside every operation, so
that tests/test_call_sequences_cpu.py can check without a GPU that the committed seeds reach the transitions the GPU
test claims to run.  Pure Python: nothing here touches torch or a device.
"""
from __future__ import annotations

import random

L = 2
P_DROP = 0.3
SEEDS = list(range(80, 96))    # 16 seeds whose sequences reach every transition tests/test_call_sequences_cpu.py checks
N_OPS = 14
GROW = 2                 # a context-growth operation asks for a window this much longer than the context's
GROW_MAX = 6             # ... up to the Trainer's T + GROW_MAX (the vocabulary holds T + GROW_MAX + GROW rows of tokens)

# row -> (H, T, B, recurrence plan, tied).  "persistent": both persistent recurrence kernels fit (K-split, odd H, a
# partly populated last cluster: tests/test_gpu_dropout.py's odd_h shape); "steps": neither fits (B = 40), every step
# is its own launch and W_hh has only its row image; "fwdonly": the forward kernel only (ZRB_REC=fwdonly), so W_hh has
# a row image for the per-timestep backward and forward slices for the persistent forward.  The lazy update defers
# only where both kernels run.
ROWS = {}
for _plan, (_H, _T, _B) in (("persistent", (257, 5, 9)), ("steps", (64, 4, 40)), ("fwdonly", (257, 5, 9))):
    for _tied in (False, True):
        ROWS[f"{_plan}-{'tied' if _tied else 'untied'}"] = (_H, _T, _B, _plan, _tied)


def vocab(T, B):
    return max(97, (T + GROW_MAX + GROW) * B + 13)


TRAIN = ("train_clip", "train_noclip", "train_host", "train_phased")
EVAL = ("eval", "ppl", "eval_cache", "fwd_eval")
DECODE = ("generate", "beam")
DROPIN = ("fwd_clip_sgd", "fwd_torch_sgd")
DYNEVAL = ("grad_stats", "dyneval_sgd", "dyneval_rms")
AVERAGE = ("avg_start", "avg_stop", "avg_enter", "avg_leave")
SWITCH = ("wd", "ed", "var", "artar", "keep_clipped", "lazy")
GROWTH = ("grow_fwd", "grow_stats")
OTHER = ("edit", "flush", "unit", "refuse")
ALPHABET = TRAIN + EVAL + DECODE + DROPIN + DYNEVAL + AVERAGE + SWITCH + GROWTH + OTHER
# evaluation-type operations: what may run inside averaged_weights()
EVAL_TYPE = EVAL + DECODE + DYNEVAL
INSIDE_OK = EVAL_TYPE + GROWTH + ("avg_leave", "flush", "unit", "refuse")
REFUSALS = ("train_in_avg", "start_in_avg", "dyneval_wide", "generate_wide", "unit_no_plan", "enter_n0",
            "stats_wide_avg", "fwd_wide_avg")


class State:
    """The generator's model of the warm twin."""

    def __init__(self, row, rng):
        self.H, self.T, self.B, self.plan, self.tied = ROWS[row]
        self.wd = rng.choice([0.0, 0.5])
        self.lazy = True
        self.pending = False          # the warm twin holds deferred updates
        self.avg_on = False
        self.avg_n = 0
        self.inside = False           # inside averaged_weights()
        self.ctx_T = self.T

    def refusals(self):
        out = ["dyneval_wide", "generate_wide"]
        if self.inside:
            out += ["train_in_avg", "start_in_avg"]
        if self.plan != "persistent":
            out.append("unit_no_plan")
        if self.avg_on and self.avg_n == 0 and not self.inside:
            out.append("enter_n0")
        if self.avg_on:
            out += ["stats_wide_avg", "fwd_wide_avg"]
        return out

    def applicable(self):
        if self.inside:
            ops = [o for o in INSIDE_OK if not (o in GROWTH and self.ctx_T + GROW > self.T + GROW_MAX)]
            return [o for o in ops if o != "unit" or self.plan == "persistent"]
        ops = []
        for o in ALPHABET:
            if o == "avg_leave" or (o == "avg_stop" and not self.avg_on) or \
                    (o == "avg_enter" and not (self.avg_on and self.avg_n > 0)):
                continue
            if o in GROWTH and self.ctx_T + GROW > self.T + GROW_MAX:
                continue
            if o == "unit" and self.plan != "persistent":
                continue
            ops.append(o)
        return ops


def flushes(name, args):
    """Whether the operation applies the warm twin's pending updates (every entry point that reads the weights does)."""
    if name in TRAIN or name in SWITCH:
        return False
    if name == "refuse":
        return args["kind"] == "enter_n0"          # averaged_weights() flushes before the library refuses the swap
    if name in GROWTH and args.get("refused"):
        return False
    return True


def _args(name, st, rng):
    w = lambda: rng.randrange(4)
    if name in ("train_clip", "train_noclip", "train_host", "train_phased", "eval", "eval_cache", "fwd_eval",
                "fwd_clip_sgd", "fwd_torch_sgd", "dyneval_sgd", "dyneval_rms", "unit"):
        return {"w": w(), "seed": rng.randrange(1 << 30)}
    if name in ("ppl", "grad_stats"):
        return {"w": w(), "w2": w()}
    if name == "generate":
        return {"Bp": rng.randint(1, st.B), "n_new": rng.randint(1, 4), "seed": rng.randrange(1 << 30)}
    if name == "beam":
        K = rng.choice([2, 3])
        return {"Bp": rng.randint(1, st.B // K), "K": K, "n_new": rng.randint(1, 3), "seed": rng.randrange(1 << 30)}
    if name == "wd":
        return {"p": rng.choice([0.0, 0.3, 0.5]), "seed": rng.randrange(1 << 40)}
    if name == "ed":
        return {"p": rng.choice([0.0, 0.2]), "seed": rng.randrange(1 << 40)}
    if name == "var":
        on = rng.random() < 0.6
        return {"on": on, "p_rec": rng.choice([0.0, 0.25]) if on else 0.0}
    if name == "artar":
        return rng.choice([{"ar": 0.0, "tar": 0.0}, {"ar": 2.0, "tar": 1.0}, {"ar": 0.5, "tar": 0.0}])
    if name in ("keep_clipped", "lazy"):
        return {"on": rng.random() < 0.5}
    if name == "edit":
        return {"i": rng.randrange(2 + 4 * L), "delta": rng.choice([-0.01, 0.02])}
    if name in GROWTH:
        return {"T": st.ctx_T + GROW, "train": rng.random() < 0.5, "seed": rng.randrange(1 << 30),
                "refused": st.avg_on}
    if name == "refuse":
        kinds = st.refusals()
        if len(kinds) > 2 and rng.random() < 0.7:
            kinds = kinds[2:]                       # mostly the refusals of the present state
        return {"kind": rng.choice(kinds), "seed": rng.randrange(1 << 30)}
    return {}


def _advance(st, name, args):
    if flushes(name, args):
        st.pending = False
    if name in TRAIN:
        st.pending = st.lazy and st.plan == "persistent"
        if st.avg_on:
            st.avg_n += 1
    elif name == "wd":
        st.wd = args["p"]
    elif name == "lazy":
        st.lazy = args["on"]
    elif name == "avg_start":
        st.avg_on, st.avg_n = True, 0
    elif name == "avg_stop":
        st.avg_on, st.avg_n = False, 0
    elif name == "avg_enter":
        st.inside = True
    elif name == "avg_leave":
        st.inside = False
    elif name in GROWTH and not args["refused"]:
        st.ctx_T = args["T"]


def sequence(row, seed, n_ops=N_OPS):
    """The operations of (row, seed): a list of dicts {op, args, and the state before it: pending, avg_on, inside,
    wd, prev}.  Ends outside averaged_weights() with a flush, after which the GPU test compares everything."""
    rng = random.Random(f"{row}/{seed}")
    st = State(row, rng)
    out = []
    prev = None
    while len(out) < n_ops:
        ops = st.applicable()
        if prev in TRAIN:                           # anything may follow a (lazy) train step
            name = rng.choices(ops, [8.0 if o == "avg_enter" else 1.0 for o in ops])[0]
        elif prev in SWITCH and len(out) >= 2 and out[-2]["op"] in TRAIN and rng.random() < 0.7 and not st.inside:
            name = rng.choice(TRAIN)                # a mode switch between two train steps
        else:
            # train often, average often, and stay a while inside averaged_weights()
            bias = {"avg_start": 0.5 if st.avg_on else 3.0, "avg_enter": 4.0, "avg_leave": 0.4}
            weights = [4.0 if o in TRAIN else bias.get(o, 1.0) for o in ops]
            name = rng.choices(ops, weights)[0]
        args = _args(name, st, rng)
        if name == "avg_enter":
            args["abi"] = len(out) % 2 == 1        # every other swap through the C ABI, which flushes by itself
        out.append(dict(op=name, args=args, pending=st.pending, avg_on=st.avg_on, inside=st.inside, wd=st.wd,
                        prev=prev, initial_wd=out[0]["initial_wd"] if out else st.wd))
        _advance(st, name, args)
        prev = name
    for name in (["avg_leave"] if st.inside else []) + ["flush"]:
        out.append(dict(op=name, args={}, pending=st.pending, avg_on=st.avg_on, inside=st.inside, wd=st.wd, prev=prev,
                        initial_wd=out[0]["initial_wd"]))
        _advance(st, name, {})
        prev = name
    return out


def describe(seq):
    return "\n".join(f"  {i:2d} {s['op']:<14s} {s['args']}" for i, s in enumerate(seq))
