"""The committed seeds of tests/test_gpu_call_sequences.py reach the transitions that test claims to run.

The GPU test compares a warm Trainer against a cold twin over seeded operation sequences (tests/_call_sequences.py).
"It passes" only means something if the sequences contain the transitions where cross-call state goes wrong; this
checks, on any machine, that over the committed seeds every one of these occurs at least once:
  * every operation, and every refusal;
  * every operation right after a lazy train step (on a row where the lazy update defers);
  * every evaluation-type operation inside averaged_weights();
  * every mode switch between two train steps, the first with weight drop on;
  * every context-growth operation while lazy updates are pending, and while averaging is on.
"""
import pytest

from tests import _call_sequences as S


def _all():
    return {(row, seed): S.sequence(row, seed) for row in S.ROWS for seed in S.SEEDS}


def _missing(want, got):
    return sorted(set(want) - set(got))


def test_every_operation_and_refusal_occurs():
    seqs = _all()
    ops = {s["op"] for seq in seqs.values() for s in seq}
    assert not _missing(S.ALPHABET, ops), _missing(S.ALPHABET, ops)
    kinds = {s["args"]["kind"] for seq in seqs.values() for s in seq if s["op"] == "refuse"}
    assert not _missing(S.REFUSALS, kinds), _missing(S.REFUSALS, kinds)


def test_every_operation_follows_a_lazy_train_step():
    after = set()
    for (row, _), seq in _all().items():
        if S.ROWS[row][3] != "persistent":
            continue
        after |= {s["op"] for s in seq if s["prev"] in S.TRAIN and s["pending"]}
    # averaged_weights() is left only from inside it, where no train step runs
    want = [o for o in S.ALPHABET if o != "avg_leave"]
    assert not _missing(want, after), _missing(want, after)


def test_every_evaluation_runs_inside_averaged_weights():
    inside = {s["op"] for seq in _all().values() for s in seq if s["inside"]}
    assert not _missing(S.EVAL_TYPE, inside), _missing(S.EVAL_TYPE, inside)


def test_every_mode_switch_sits_between_train_steps_with_weight_drop_on():
    seen = set()
    for seq in _all().values():
        for i in range(1, len(seq) - 1):
            a, s, b = seq[i - 1], seq[i], seq[i + 1]
            if s["op"] in S.SWITCH and a["op"] in S.TRAIN and a["wd"] > 0 and b["op"] in S.TRAIN:
                seen.add(s["op"])
    assert not _missing(S.SWITCH, seen), _missing(S.SWITCH, seen)


@pytest.mark.parametrize("flag", ["pending", "avg_on"])
def test_every_context_growth_meets_pending_updates_and_averaging(flag):
    seen = set()
    for (row, _), seq in _all().items():
        if flag == "pending" and S.ROWS[row][3] != "persistent":
            continue
        seen |= {s["op"] for s in seq if s["op"] in S.GROWTH and s[flag]}
    assert not _missing(S.GROWTH, seen), _missing(S.GROWTH, seen)


def test_sequences_are_reproducible_and_follow_the_rules():
    for (row, seed), seq in _all().items():
        assert seq == S.sequence(row, seed), "a seed must replay the same sequence"
        assert seq[-1]["op"] == "flush" and not seq[-1]["inside"]
        for s in seq:
            assert not (s["inside"] and (s["op"] in S.TRAIN or s["op"] in S.SWITCH or s["op"] in S.DROPIN))
            if s["op"] in S.GROWTH:
                assert s["args"]["refused"] == s["avg_on"]
