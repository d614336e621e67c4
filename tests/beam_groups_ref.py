"""TEST INFRASTRUCTURE. Grouped beam search (rwkv_b200_beam_search_groups) restated on the host for tests/test_beam_groups_host.py and
tests/test_gpu_beam_groups.py: G searches of beam_ref's rules run in lockstep, one step of every running group, then one advance of all
the beams they took together, as the device loop runs one pass for every group."""
import beam_ref as br


def search_groups(roots, width, max_tokens, stops, candidates, advance_all):
    """roots[g]: group g's root handle; candidates(handle) -> [(token, lp)]; advance_all(moves) -> handles, where moves[g] is None for
    a group that did not step, else [(parent handle, token)] of the beams it took (possibly empty), and the result lists the new
    handles in the same shape. Returns per group (pool, live, last taken) as beam_ref.search does; a group with max_tokens 0 gives
    ([], [], [])."""
    G = len(roots)
    pool = [[] for _ in range(G)]
    live = [[(0.0, [], roots[g])] if max_tokens[g] > 0 else [] for g in range(G)]
    last = [[] for _ in range(G)]
    running = [max_tokens[g] > 0 for g in range(G)]
    step = 0
    while any(running):
        taken = [None] * G
        for g in range(G):
            if not running[g]:
                continue
            t, finished = br.walk([candidates(h) for _, _, h in live[g]], [s for s, _, _ in live[g]], width, len(pool[g]), stops)
            pool[g] += [(sc, live[g][b][1] + [tok]) for b, tok, sc in finished]
            taken[g] = t
        handles = advance_all([None if t is None else [(live[g][b][2], tok) for b, tok, _ in t] for g, t in enumerate(taken)])
        for g in range(G):
            if taken[g] is None:
                continue
            live[g] = [(sc, live[g][b][1] + [tok], h) for (b, tok, sc), h in zip(taken[g], handles[g])]
            if live[g]:
                last[g] = live[g]
            running[g] = bool(live[g]) and len(pool[g]) < width and step + 1 < max_tokens[g]
        step += 1
    return [(pool[g], live[g], last[g]) for g in range(G)]


def one_by_one(advance):
    """advance_all from a per-beam advance(handle, token)."""
    return lambda moves: [None if m is None else [advance(h, t) for h, t in m] for m in moves]


def results_groups(found, length_penalty, n_best):
    """Rules 4 and 5 per group: [[(tokens, score, finished)]]."""
    return [br.results(pool, live, length_penalty[g], n_best) for g, (pool, live, _) in enumerate(found)]
