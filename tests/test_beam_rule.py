"""calm_b200_decode_beam's rule (include/calm_b200.h) as tests/beam_ref.py restates it, checked on hand-worked cases and
against a brute-force search over every continuation of a toy distribution when the beam is as wide as the paths."""
import itertools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import beam_ref as br  # noqa: E402

f32 = np.float32


def lists(*rows):
    """One step's (ids, lps) from rows of (id, lp) pairs."""
    return np.asarray([[i for i, _ in r] for r in rows], np.int32), np.asarray([[lp for _, lp in r] for r in rows], np.float32)


def tokens(out):
    return [h[0].tolist() for h in out["hyps"]]


def test_candidate_count_leaves_num_beams_non_stop_candidates():
    assert br.n_candidates(1, 0) == 2 and br.n_candidates(3, 0) == 6 and br.n_candidates(2, 4) == 10 and br.n_candidates(10, 1) == 20


def test_a_stop_past_walk_position_num_beams_is_skipped():
    # B 2, stop 9, K 4.  Step 0: beams [1] (S -0.125) and [2] (S -0.5); the stop at q 1 finishes [9].
    s0 = lists([(1, -0.125), (9, -0.25), (2, -0.5), (3, -1.0)])
    # step 1: c = -0.25 (b0 5), -0.375 (b0 stop, q 1: finishes), -0.5625 (b1 stop, q 2: skipped), -1.5 (b1 6)
    s1 = lists([(5, -0.125), (9, -0.25), (7, -4.0), (8, -5.0)], [(9, -0.0625), (6, -1.0), (7, -6.0), (8, -7.0)])
    out = br.replay([s0, s1], 2, stop=[9], length_penalty=0.0, early_stopping=1)
    assert [b for b, _, _ in out["back"][1]] == [0, 1] and [t for _, t, _ in out["back"][1]] == [5, 6]
    # pool: [9] (-0.25) and [1, 9] (-0.375), full after step 1: done
    assert out["steps"] == 2
    assert tokens(out) == [[9], [1, 9]]
    assert [h[2] for h in out["hyps"]] == [f32(-0.25), f32(-0.375)]
    assert out["anc"][:2, :2].tolist() == [[0, 0], [0, 1]]
    # early_stopping 0: worst -0.375 < S_best -0.25, so not done; after the last step [1, 5] (-0.25) evicts [1, 9] and
    # [2, 6] (-1.5) stays out; [9] and [1, 5] tie, [9] was added first
    out = br.replay([s0, s1], 2, stop=[9], length_penalty=0.0)
    assert out["steps"] == 2 and tokens(out) == [[9], [1, 5]]


def test_ties_go_to_the_lower_beam_then_the_lower_rank():
    s0 = lists([(3, -1.0), (4, -1.0), (5, -2.0), (6, -2.0)])
    s1 = lists([(7, -1.0), (8, -1.0), (1, -3.0), (2, -3.0)], [(8, -1.0), (7, -1.0), (1, -3.0), (2, -3.0)])
    out = br.replay([s0, s1], 2)
    assert out["beams"][1] == [[3], [4]]
    assert out["back"][1] == [(0, 7, f32(-1.0)), (0, 8, f32(-1.0))]
    assert tokens(out) == [[3, 7], [3, 8]]  # equal scores: the earlier added first
    assert [h[2] for h in out["hyps"]] == [f32(-1.0), f32(-1.0)]  # -2 / norm[2] = 2


def test_pool_evicts_the_earliest_of_equal_worst_scores():
    p = br.Pool(2)
    p.add(f32(-1), [1], [-1], f32(-1))
    p.add(f32(-1), [2], [-1], f32(-1))
    p.add(f32(-1), [3], [-1], f32(-1))  # not strictly better than the worst: stays out
    assert [h[2] for h in p.items] == [[1], [2]]
    p.add(f32(-0.5), [4], [-0.5], f32(-0.5))  # [1] and [2] tie as worst: [1] was added first and leaves
    assert [h[2] for h in p.items] == [[2], [4]]
    assert [h[2] for h in p.ordered()] == [[4], [2]]
    p.add(f32(-0.5), [5], [-0.5], f32(-0.5))  # evicts [2]; [4] and [5] tie and keep their order
    assert [h[2] for h in p.ordered()] == [[4], [5]]


def early_case():
    """B 1, stop 9, K 2, length_penalty 2.  Step 0: [1], S -1.  Step 1: the stop finishes [1, 9], raw -1.5, score -1.5 /
    norm[1] = -1.5; the beam is [1, 2], S -2.  Step 2: [1, 2, 4], S -2.25; it enters the pool after max_new 3 steps with
    -2.25 / 9 = -0.25 and evicts [1, 9]."""
    s0 = lists([(1, -1.0), (9, -3.0)])
    s1 = lists([(9, -0.5), (2, -1.0)])
    s2 = lists([(4, -0.25), (9, -3.0)])
    return [s0, s1, s2]


def test_early_stopping_1_stops_once_the_pool_is_full():
    out = br.replay(early_case(), 1, stop=[9], length_penalty=2.0, early_stopping=1)
    assert out["steps"] == 2 and tokens(out) == [[1, 9]] and out["hyps"][0][2] == f32(-1.5)


def test_early_stopping_0_continues_past_a_full_pool():
    # after step 1 the pool is full, but worst -1.5 < S_best / norm[2] = -2 / 4: not done; after step 2, -1.5 < -2.25 / 9
    out = br.replay(early_case(), 1, stop=[9], length_penalty=2.0, early_stopping=0)
    assert out["steps"] == 3 and tokens(out) == [[1, 2, 4]]
    assert out["hyps"][0][2] == f32(f32(-2.25) / f32(9.0))
    assert out["hyps"][0][1].tolist() == [-1.0, -1.0, -0.25] and br.fsum(out["hyps"][0][1]) == f32(-2.25)


@pytest.mark.parametrize("penalty", [0.0, 1.0, 2.0])
def test_length_penalty_divides_by_the_length_to_its_power(penalty):
    steps = [lists([(1, -0.5), (2, -2.0)])] + [lists([(3, -0.5), (2, -2.0)])] * 2
    out = br.replay(steps, 1, length_penalty=penalty)
    assert tokens(out) == [[1, 3, 3]]
    assert out["hyps"][0][2] == f32(f32(-1.5) / f32(3.0 ** penalty))
    # a stop at step j is normalised by the j tokens before it
    out = br.replay([lists([(1, -0.5), (9, -2.0)]), lists([(9, -0.25), (2, -2.0)])], 1, stop=[9], length_penalty=penalty, early_stopping=1)
    assert tokens(out) == [[1, 9]] and out["hyps"][0][2] == f32(-0.75)


def test_a_stop_at_step_0_is_normalised_as_length_1():
    out = br.replay([lists([(9, -0.5), (1, -1.0)])], 1, stop=[9], length_penalty=2.0, early_stopping=1, max_new=4)
    assert out["steps"] == 1 and tokens(out) == [[9]] and out["hyps"][0][2] == f32(-0.5)


def test_norm_table_is_pow_in_double_rounded_once():
    t = br.norm_table(5, 1.3)
    assert t[1:] == [f32(float(L) ** 1.3) for L in range(1, 6)] and all(type(x) is np.float32 for x in t)


def toy(history, V, rng_seed):
    """The toy model's log-probabilities of the V real tokens after `history` (float32)."""
    r = np.random.default_rng(hash((rng_seed,) + tuple(history)) % (1 << 32))
    z = r.normal(size=V)
    return (z - np.log(np.exp(z).sum())).astype(np.float32)


@pytest.mark.parametrize("seed,length_penalty", [(1, 1.0), (2, 0.0), (3, 2.5)])
def test_a_beam_as_wide_as_the_paths_is_exhaustive(seed, length_penalty):
    """V = 3 real tokens over 2 steps: 9 paths, B = 9 (K = 18).  The lists are each row's real tokens in rank order, then
    filler ids whose log-probability (-1e30) keeps them last; every path survives to the end, and the output is every
    path by its score."""
    V, B, T = 3, 9, 2
    K = br.n_candidates(B, 0)
    filler = np.float32(-1e30)

    def row(history):
        lp = toy(history, V, seed)
        order = np.lexsort((np.arange(V), -lp.astype(np.float64)))
        ids = list(order) + list(range(V, K))
        return ids, [lp[i] for i in order] + [filler] * (K - V)

    steps, live = [], [[]]  # each step's rows follow the beams the rule made of the steps before it
    for j in range(T):
        rows = [row(h) for h in live]
        steps.append((np.asarray([r[0] for r in rows], np.int32), np.asarray([r[1] for r in rows], np.float32)))
        live = br.replay(steps, B, length_penalty=length_penalty, max_new=T)["live"]
    out = br.replay(steps, B, length_penalty=length_penalty)
    norm = br.norm_table(T, length_penalty)
    want = []
    for path in itertools.product(range(V), repeat=T):
        lps = [toy(path[:i], V, seed)[path[i]] for i in range(T)]
        want.append((br.fsum(lps) / norm[T], list(path)))
    want.sort(key=lambda x: -float(x[0]))
    assert [h[0].tolist() for h in out["hyps"]] == [p for _, p in want]
    assert [h[2] for h in out["hyps"]] == [s for s, _ in want]
