"""Seeded interleavings of every entry point on one context against a serial replay (tests/interleave.py). Every other engine test
starts from a fresh context and exercises one feature; here an odd-length generate is followed by a longer rwkv_eval_sequence that
regrows the scratch, a graph-replayed rwkv_eval, a generate that keeps its counts, a clone, a toggle -- and after every op the
context's state, logits, validity, counts and automaton state must equal those of feeding the same tokens one at a time through
rwkv_eval on a separate plain context, bit for bit. Passes that take the tensor cores are held to the end-to-end bars instead, and
the replay then adopts the context's bytes."""
import os
import time

import numpy as np
import pytest

import interleave as il
from conftest import VERSIONS, model_path

pytestmark = pytest.mark.gpu

N_OPS, B = 80, 5
FILES = [(ver, fmt) for ver in VERSIONS for fmt in ("FP32", "Q5_1")] + [("6v0-3m", "FP16")]
LARGE = [("rwkv6-small", "Q5_1", 1.5e-1), ("rwkv7-small", "FP16", 2e-2), ("rwkv5-small", "Q4_0", 1.5e-1)]    # the bars of test_gpu_parity.py after long prompts
_env = os.environ.get("RWKV_INTERLEAVE_SEEDS")
SEEDS = [int(s) for s in _env.split(",")] if _env else None      # None: two fixed seeds per file, 0 .. 21 over the eleven files
COVER = dict(single=dict(kinds=set(), pairs=set()), batch=dict(kinds=set(), pairs=set()), lines=[], schedules=0, ops=0, t0=time.time())


def seeds_of(i):
    return SEEDS if SEEDS is not None else [2 * i, 2 * i + 1]


def record(group, label, stats):
    COVER[group]["kinds"] |= set(stats["ops"])
    COVER[group]["pairs"] |= stats["pairs"]
    COVER["schedules"] += 1
    COVER["ops"] += sum(stats["ops"].values())
    COVER["lines"].append(f"{label}: {sum(stats['ops'].values())} ops, {stats['graph_ops']} launched a CUDA graph, {stats['rebases']} re-based")


def anchor(path):
    """The shadow must not be self-referential: one more token from each sequence's final state, against the numpy oracle run over
    that sequence's whole token history from a fresh state."""
    def check(r):
        import rwkv_oracle as ro
        oracle = ro.OracleModel(path)
        for s in r.cur.sh.seqs[:2]:         # of a batch, the first two sequences: the oracle takes seconds per long history
            want, _ = oracle.eval_sequence(s.history + [10])
            got = r.drv.step(s.state, 10)[1]
            assert np.abs(got - want).max() <= 1e-3, (len(s.history), float(np.abs(got - want).max()))
    return check


def run(lib, path, schedule, seed, label, group, **kw):
    drv = il.LibDriver(lib, path)
    try:
        stats = il.run_schedule(drv, schedule, label=label, seed=seed, where=__file__, **kw)
    finally:
        drv.close()
    record(group, f"{label} seed {seed}", stats)
    return stats


@pytest.mark.parametrize("i", range(len(FILES)), ids=["-".join(f) for f in FILES])
def test_single_context_bit_exact(lib, i):
    ver, fmt = FILES[i]
    for seed in seeds_of(i):
        run(lib, model_path(ver, fmt), il.make_schedule(seed, il.SINGLE_KINDS, N_OPS), seed, f"single {ver} {fmt}", "single",
            on_end=anchor(model_path(ver, fmt)) if fmt == "FP32" else None)


@pytest.mark.parametrize("i", range(len(FILES)), ids=["-".join(f) for f in FILES])
def test_batch_context_bit_exact(lib, i):
    ver, fmt = FILES[i]
    for seed in seeds_of(i):
        run(lib, model_path(ver, fmt), il.make_schedule(seed, il.BATCH_KINDS, N_OPS, B=B), seed, f"batch {ver} {fmt}", "batch", B=B,
            on_end=anchor(model_path(ver, fmt)) if fmt == "FP32" else None)


@pytest.mark.parametrize("ver,fmt", [("5v2-730K", "Q5_1"), ("6v0-3m", "FP32"), ("7v0-834K", "Q5_1")])
def test_batch_context_tensor_cores_off_stays_bit_exact_at_any_sum(lib, ver, fmt):
    seed = 100 + VERSIONS.index(ver)
    run(lib, model_path(ver, fmt), il.make_schedule(seed, il.BATCH_KINDS, 50, B=B, large=True, tc_toggle=False), seed, f"batch tc-off {ver} {fmt}", "batch",
        B=B, tc=False)


def test_single_context_tensor_cores_off_stays_bit_exact_at_any_length(lib):
    run(lib, model_path("6v0-3m", "Q5_1"), il.make_schedule(200, il.SINGLE_KINDS, 50, large=True, tc_toggle=False), 200, "single tc-off 6v0-3m Q5_1", "single",
        tc=False)


@pytest.fixture(scope="module")
def synthetic(tmp_path_factory):
    import synthetic_model as sm
    d = tmp_path_factory.mktemp("interleave")
    paths = {}
    for preset, fmt, _ in LARGE:
        paths[preset] = str(d / f"{preset}-{fmt}.bin")
        sm.write_direct(paths[preset], preset, fmt, seed=11)
    return paths


@pytest.mark.parametrize("preset,fmt,tol", LARGE)
def test_large_passes_rebase(lib, synthetic, preset, fmt, tol):
    """Passes of 32 .. 300 tokens take the tensor cores: held to the end-to-end bar, then the replay adopts the context's bytes and
    every later op is bit-exact again. rwkv6-small takes the LoRA fold in its single-token passes and not in the others, so the two
    routes alternate on one state."""
    if preset == "rwkv6-small":
        import ggml_file as gf
        assert lib.library.rwkv_b200_v6_lora_fold_supported(512, 64, gf.TYPE_IDS[fmt], 32, gf.TYPE_IDS[fmt], 64)
    seed = 300 + len(preset) + len(fmt)
    stats = run(lib, synthetic[preset], il.make_schedule(seed, il.SINGLE_KINDS, 60, large=True), seed, f"large single {preset} {fmt}", "single", tol=tol)
    assert stats["rebases"] > 0
    stats = run(lib, synthetic[preset], il.make_schedule(seed, il.BATCH16_KINDS, 40, large=True, B=16), seed, f"large batch-16 {preset} {fmt}", "batch",
                B=16, tol=tol)
    assert stats["rebases"] > 0


# ---- teeth: the real library misused in one way; the harness must report it within the schedule -----------------------------------

class KeepDropped(il.LibDriver):
    def keep_flag(self, g):
        return False if isinstance(g["keep"], bool) else None


class RaggedShifted(il.LibDriver):
    """Hands sequence b's tokens to sequence b + 1: the counts rotate by one."""
    def batch_eval_ragged(self, c, tokens, counts, want):
        return super().batch_eval_ragged(c, tokens, counts[-1:] + counts[:-1], want) if sum(counts) else super().batch_eval_ragged(c, tokens, counts, want)


class SetStateDropped(il.LibDriver):
    dropped = False

    def batch_set_state(self, c, seq, state, mem):
        if not self.dropped:
            self.dropped = True
            return True
        return super().batch_set_state(c, seq, state, mem)


class StaleLogits(il.LibDriver):
    """Reports the logits it fetched before a pass without the head as current."""
    def __init__(self, *a):
        super().__init__(*a)
        self.seen = {}

    def batch_get_logits(self, c, seq, mem):
        ok, lg = super().batch_get_logits(c, seq, mem)
        if ok:
            self.seen[seq] = lg
            return ok, lg
        self.lib.rwkv_get_last_error(c)
        return (True, self.seen[seq]) if seq in self.seen else (ok, lg)


class ChunkTruncated(il.LibDriver):
    def eval_chunks(self, c, tokens, chunk, state, out, logits, mem):
        return super().eval_chunks(c, tokens[:-1] if len(tokens) > 1 else tokens, chunk, state, out, logits, mem)


@pytest.mark.parametrize("driver,batch", [(KeepDropped, False), (KeepDropped, True), (RaggedShifted, True), (SetStateDropped, True), (StaleLogits, True),
                                          (ChunkTruncated, False)], ids=lambda v: getattr(v, "__name__", str(v)))
def test_a_misused_library_is_reported_within_the_schedule(lib, driver, batch):
    path = model_path("6v0-3m", "Q5_1")
    caught = 0
    for seed in range(4):
        drv = driver(lib, path)
        try:
            sched = il.make_schedule(seed, il.BATCH_KINDS, N_OPS, B=B) if batch else il.make_schedule(seed, il.SINGLE_KINDS, N_OPS)
            with pytest.raises(AssertionError, match=r"op \d+ \(\w+\) failed"):
                il.run_schedule(drv, sched, B=B if batch else 0, label=driver.__name__, seed=seed, where=__file__)
            caught += 1
        except pytest.fail.Exception:
            pass                     # this seed's schedule happens not to depend on the broken rule
        finally:
            drv.close()
        if caught:
            break
    assert caught, driver.__name__


def test_coverage(request, lib):
    """Every op kind and every ordered pair of kinds ran, single and batch. Prints per schedule how many ops launched a CUDA graph
    (single-token replays and generation loops, from rwkv_b200_graph_launch_count) and how many re-based. A run of part of the file
    (-k, a node id) or with other seeds skips it."""
    n_items = 2 * len(FILES) + 3 + 1 + len(LARGE) + 6 + 1
    if sum(i.fspath == request.node.fspath for i in request.session.items) < n_items or SEEDS is not None:
        pytest.skip("only part of the file, or another seed set, was selected")
    import subprocess
    for line in COVER["lines"]:
        print(line)
    for group, kinds in (("single", il.SINGLE_KINDS), ("batch", il.BATCH_KINDS)):
        assert COVER[group]["kinds"] == set(kinds), set(kinds) - COVER[group]["kinds"]
        missing = {(a, b) for a in kinds for b in kinds} - COVER[group]["pairs"]
        assert not missing, sorted(missing)
    n_pairs = len(COVER["single"]["pairs"]) + len(COVER["batch"]["pairs"])
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    graph_ops = sum(int(line.split(" ops, ")[1].split(" ")[0]) for line in COVER["lines"])
    rebases = sum(int(line.split(", ")[-1].split(" ")[0]) for line in COVER["lines"])
    assert graph_ops > 0 and rebases > 0
    print(f"{COVER['schedules']} schedules, {COVER['ops']} ops, {n_pairs} distinct (kind -> kind) pairs; {graph_ops} ops launched a CUDA graph, "
          f"{rebases} re-bases; {time.time() - COVER['t0']:.0f} s wall on {card}")
