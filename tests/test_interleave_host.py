"""The interleaving harness (tests/interleave.py) without a GPU: the schedule generator is deterministic and covers what it promises,
every default schedule passes on the toy engine, and the toy engine with one bookkeeping rule broken is reported with the failing op."""
import ast
import re
from collections import Counter

import numpy as np
import pytest

import generate_ref as gr
import interleave as il

N_OPS, B = 80, 5
SINGLE_SEEDS = list(range(22))      # the GPU file gives each of its 11 model files two of them
BATCH_SEEDS = list(range(22))


def single(seed):
    return il.make_schedule(seed, il.SINGLE_KINDS, N_OPS)


def batch(seed):
    return il.make_schedule(seed, il.BATCH_KINDS, N_OPS, B=B)


def test_generator_is_deterministic_and_prints_as_a_literal():
    for make in (single, batch):
        s = make(3)
        assert repr(s) == repr(make(3)) and repr(s) != repr(make(4))
        assert ast.literal_eval(repr(s)) == s


@pytest.mark.parametrize("make,kinds,seeds", [(single, il.SINGLE_KINDS, SINGLE_SEEDS), (batch, il.BATCH_KINDS, BATCH_SEEDS)])
def test_every_kind_per_schedule_and_every_pair_over_the_default_seeds(make, kinds, seeds):
    pairs = set()
    for seed in seeds:
        s = make(seed)
        assert len(s) == N_OPS and {k for k, _ in s} == set(kinds), seed
        pairs |= il.pairs_of(s)
    assert pairs == {(a, b) for a in kinds for b in kinds}
    assert il.seeds_for_all_pairs(kinds, N_OPS) <= len(seeds)
    first = set()
    for seed in range(il.seeds_for_all_pairs(kinds, N_OPS)):
        first |= il.pairs_of(make(seed))
    assert first == pairs


def test_automata_have_three_to_six_states_and_one_dead_end():
    for name in il.DFAS:
        t = il.dfa_table(name, 256)
        assert 3 <= t.shape[0] <= 6, (name, t.shape)
    assert any(not (il.dfa_table("ab", 256)[s] != il.bd.DEAD).any() for s in range(il.dfa_table("ab", 256).shape[0]))


@pytest.mark.parametrize("seed", SINGLE_SEEDS)
def test_single_schedules_pass_on_the_toy_engine(seed):
    stats = il.run_schedule(il.ToyDriver(), single(seed), label="toy", seed=seed)
    assert sum(stats["ops"].values()) == N_OPS


@pytest.mark.parametrize("seed", BATCH_SEEDS)
def test_batch_schedules_pass_on_the_toy_engine(seed):
    stats = il.run_schedule(il.ToyDriver(), batch(seed), B=B, label="toy batch", seed=seed)
    assert sum(stats["ops"].values()) == N_OPS


def test_large_pass_schedules_pass_on_the_toy_engine():
    il.run_schedule(il.ToyDriver(), il.make_schedule(1, il.SINGLE_KINDS, N_OPS, large=True), tol=0.0, label="toy large", seed=1)
    il.run_schedule(il.ToyDriver(), il.make_schedule(1, il.BATCH16_KINDS, 40, large=True, B=16), B=16, tol=0.0, label="toy large batch", seed=1)
    il.run_schedule(il.ToyDriver(), il.make_schedule(2, il.BATCH_KINDS, N_OPS, large=True, tc_toggle=False, B=B), B=B, tc=False, label="toy tc off", seed=2)


def test_a_printed_schedule_replays():
    s = single(5)
    want = il.run_schedule(il.ToyDriver(), s)
    got = il.run_schedule(il.ToyDriver(), ast.literal_eval(repr(s)))
    assert got["ops"] == want["ops"] and got["pairs"] == want["pairs"]


SINGLE_DEFECTS = ["parity", "stale_graph", "keep_counts", "stop_advances", "valid_sticky", "profile_noop", "clone_counts"]
BATCH_DEFECTS = ["idle_state", "frozen_logits", "keep_counts", "stop_advances", "valid_sticky"]


@pytest.mark.parametrize("defect,is_batch", [(d, False) for d in SINGLE_DEFECTS] + [(d, True) for d in BATCH_DEFECTS])
def test_each_defect_is_caught_and_the_message_replays_it(defect, is_batch):
    assert set(SINGLE_DEFECTS) | set(BATCH_DEFECTS) == set(il.DEFECTS)
    caught = 0
    for seed in (BATCH_SEEDS if is_batch else SINGLE_SEEDS):
        s = batch(seed) if is_batch else single(seed)
        try:
            il.run_schedule(il.ToyDriver(defect), s, B=B if is_batch else 0, label=defect, seed=seed)
        except AssertionError as e:
            msg = str(e)
            m = re.search(r"seed (\d+): op (\d+) \((\w+)\) failed", msg)
            assert m and int(m.group(1)) == seed and "interleave.py" in msg, msg
            i, kind = int(m.group(2)), m.group(3)
            assert s[i][0] == kind
            literal = ast.literal_eval(msg[msg.index("run_schedule(driver, ") + len("run_schedule(driver, "):msg.rindex(")")])
            assert literal == s[:i + 1]
            if not caught:      # the literal reproduces the failure on its own, and passes on the sound engine
                with pytest.raises(AssertionError, match=rf"op {i} \({kind}\)"):
                    il.run_schedule(il.ToyDriver(defect), literal, B=B if is_batch else 0)
                il.run_schedule(il.ToyDriver(), literal, B=B if is_batch else 0)
            caught += 1
    assert caught >= 1, defect


def test_shadow_generate_agrees_with_the_host_loop_of_generate_ref():
    """Shadow.generate against generate_ref.host_generate, both on the toy model: host_generate drives a sample / eval_token pair, here
    the toy engine's."""
    drv = il.ToyDriver()

    class ToyLib:      # the two calls host_generate makes, on a toy context
        class library:
            @staticmethod
            def rwkv_b200_sample(c, temperature, top_p, u, ids, vals, n, tok):
                ok, t = drv.sample(c, temperature, top_p, u, {int(ids[i]): float(vals[i]) for i in range(n)})
                tok._obj.value = t
                return ok

            @staticmethod
            def rwkv_b200_eval_resident(c, toks, n, want, out):
                return drv.eval_resident(c, [int(toks[i]) for i in range(n)], want, False, None)[0]

    rng = np.random.RandomState(7)
    for case in range(12):
        c = drv.new_context()
        sh = il.Shadow(drv)
        prompt = [int(t) for t in rng.randint(0, 256, 4)]
        drv.eval_resident(c, prompt, True, False, None)
        sh.advance(0, prompt, True)
        n = int(rng.randint(1, 10))
        us = [float(u) for u in rng.random_sample(n)]
        stops = sh.stops(0, [0, 2]) if case % 2 else []
        temperature, top_p, pres, freq = [(0.0, 1.0, 0.0, 0.0), (1.0, 0.9, 0.4, 0.3), (1.5, 0.5, 0.0, 0.3)][case % 3]
        counts = Counter()
        want = gr.host_generate(ToyLib, c, n, temperature, top_p, pres, freq, us, stops, counts)
        got, _ = sh.generate(0, n, temperature, top_p, pres, freq, False, us, stops)
        assert got == want and sh.seqs[0].counts == counts and sh.seqs[0].state == c.state[0]
