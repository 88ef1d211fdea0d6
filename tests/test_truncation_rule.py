"""The top-k / top-p rule of calm_b200_decode_sample_queue_truncated (include/calm_b200.h), restated with numpy and
Python integers, and checked against a brute-force sort-and-accumulate in exact rationals.  The GPU tests import the
restatement (`kept`, `truncate`, `boundary_slack`).

Rank order: allowed tokens (l != -inf) by logit descending, equal logits lowest id first.  Mass: m(v) =
floor(expf((l(v) - M) / T) * 2^40).  top_k K (0 off) keeps the first K ranks; top_p P (1 off) keeps the shortest prefix
of that set, at least one token, whose mass sum reaches ceil(Z P), Z the set's mass, P the fp32 value taken exactly."""
import math
from fractions import Fraction

import numpy as np
import pytest

SCALE = 1 << 40


def rank_order(l):
    """The allowed ids of row l in rank order."""
    l = np.asarray(l, np.float32)
    ids = np.nonzero(l != -np.inf)[0]
    return ids[np.lexsort((ids, -l[ids].astype(np.float64)))]


def masses(l, temperature):
    """m(v) for every id as uint64 (0 where l is -inf), from float32 expf((l - M) / T) as numpy forms it."""
    l = np.asarray(l, np.float32)
    mx = l.max()
    with np.errstate(invalid="ignore", over="ignore"):
        q = np.exp(((l - mx) / np.float32(temperature)).astype(np.float32)).astype(np.float32)
    q = np.where(l == -np.inf, np.float32(0), q)
    return np.floor(q.astype(np.float64) * SCALE).astype(np.uint64)


def target(z, top_p):
    """ceil(z * P) for the fp32 P, exactly: P = N 2^-149 with N an integer."""
    n = int(float(np.float32(top_p)) * 2.0 ** 149)
    return (z * n + (1 << 149) - 1) >> 149


def kept(l, temperature, top_k, top_p, m=None):
    """The number of leading ranks the rule keeps, and the rank order."""
    order = rank_order(l)
    n = len(order)
    if top_k > 0:
        n = min(n, top_k)
    if np.float32(top_p) < 1:
        m = masses(l, temperature) if m is None else m
        cum = np.cumsum(m[order[:n]], dtype=np.uint64)
        t = target(int(cum[-1]), top_p)
        n = int(np.searchsorted(cum, np.uint64(t), side="left")) + 1
    return n, order


def truncate(l, temperature, top_k, top_p):
    """Row l with -inf at every id the rule drops."""
    n, order = kept(l, temperature, top_k, top_p)
    out = np.full(len(l), -np.inf, np.float32)
    out[order[:n]] = np.asarray(l, np.float32)[order[:n]]
    return out


def boundary_slack(l, temperature, top_k, top_p, n_got):
    """Whether keeping n_got ranks instead of the rule's n is explained by expf differing by an ulp: the cumulative mass
    at the two prefix lengths lies within that bound of the target.  Exact for top-k alone."""
    n, order = kept(l, temperature, top_k, top_p)
    if n == n_got:
        return True
    if np.float32(top_p) >= 1 or abs(n - n_got) > 64:
        return False
    m = masses(l, temperature)
    k = len(order) if top_k <= 0 else min(top_k, len(order))
    cum = np.cumsum(m[order[:k]].astype(object))
    z = int(cum[-1])
    t = target(z, top_p)
    tol = 4 * (z >> 23) + 4 * k  # an ulp of each expf, and the floor
    lo, hi = min(n, n_got), max(n, n_got)
    return abs(int(cum[lo - 1]) - t) <= tol or abs(int(cum[hi - 2]) - t) <= tol


def brute(l, temperature, top_k, top_p):
    """The kept ids by sorting pairs and accumulating in exact rationals."""
    l = [float(x) for x in np.asarray(l, np.float32)]
    m = masses(l, temperature)
    items = sorted(((-x, i) for i, x in enumerate(l) if x != -math.inf))
    if top_k > 0:
        items = items[:top_k]
    if float(np.float32(top_p)) < 1:
        z = sum(int(m[i]) for _, i in items)
        goal = Fraction(z) * Fraction(float(np.float32(top_p)))
        acc, out = 0, []
        for x, i in items:
            out.append((x, i))
            acc += int(m[i])
            if acc >= goal:
                break
        items = out
    return sorted(i for _, i in items)


def check(l, temperature, top_k, top_p):
    n, order = kept(l, temperature, top_k, top_p)
    assert sorted(order[:n].tolist()) == brute(l, temperature, top_k, top_p)
    assert n >= 1
    row = truncate(l, temperature, top_k, top_p)
    assert np.isfinite(row).sum() == n
    return n, order


def test_key_order_and_masses():
    l = np.asarray([0.0, -1.0, 0.0, -np.inf, 3.0], np.float32)
    assert rank_order(l).tolist() == [4, 0, 2, 1]
    m = masses(l, 1.0)
    assert int(m[4]) == SCALE and int(m[3]) == 0


def test_ties_across_the_top_k_boundary():
    l = np.asarray([1, 5, 3, 3, 3, 3, 0, 3], np.float32)
    n, order = check(l, 1.0, 3, 1.0)
    assert order[:n].tolist() == [1, 2, 3]  # the lowest ids of the tie group
    n, order = check(l, 1.0, 6, 1.0)
    assert sorted(order[:n].tolist()) == [1, 2, 3, 4, 5, 7]


def test_tie_group_straddles_the_nucleus_boundary():
    l = np.asarray([0.0] * 10 + [2.0], np.float32)
    for p in (0.5, 0.7, 0.9, 0.95):
        n, order = check(l, 1.0, 0, p)
        assert order[0] == 10 and order[1:n].tolist() == list(range(n - 1))


def test_target_hit_exactly():
    for count, j in ((8, 3), (16, 5), (4, 1), (32, 31)):
        l = np.zeros(count + 5, np.float32)
        l[count:] = -50.0  # zero-mass tail at T = 1
        p = j / count  # exactly representable
        n, order = check(l, 1.0, 0, p)
        assert n == j, (count, j, n)  # >=, not >: the prefix stops where the sum equals the target


def test_zero_mass_tails_and_smallest_p():
    l = np.asarray([10.0, -100.0, -200.0, -300.0], np.float32)
    assert check(l, 1.0, 0, 0.999)[0] == 1  # the tail has mass 0: never part of the nucleus
    tiny = np.nextafter(np.float32(0), np.float32(1))
    for row in (l, np.zeros(50, np.float32)):
        assert check(row, 1.0, 0, tiny)[0] == 1
    assert target(SCALE, tiny) == 1


def test_k_beyond_the_allowed_set_and_all_but_one_masked():
    l = np.full(100, -np.inf, np.float32)
    l[[3, 40, 77]] = [1.0, 2.0, 2.0]
    assert check(l, 1.0, 50, 1.0)[0] == 3
    assert check(l, 0.6, 200, 0.9)[0] >= 2
    one = np.full(64, -np.inf, np.float32)
    one[17] = -4.0
    for k, p in ((1, 1.0), (5, 0.5), (0, 0.01)):
        n, order = check(one, 1.0, k, p)
        assert n == 1 and order[0] == 17


def test_nucleus_is_normalised_over_the_top_k_set():
    # two tokens of equal mass above many small ones: over all tokens P = 0.5 needs one or two of the big ones and
    # some small; over the top-2 set it needs exactly one
    l = np.asarray([5.0, 5.0] + [4.0] * 20, np.float32)
    n_k, _ = check(l, 1.0, 2, 0.5)
    n_all, _ = check(l, 1.0, 0, 0.5)
    assert n_k == 1 and n_all > 2


def test_masses_follow_the_temperature():
    l = np.asarray([0.0, -1.0, -2.0, -3.0, -4.0], np.float32)
    assert check(l, 0.25, 0, 0.9)[0] < check(l, 4.0, 0, 0.9)[0]


@pytest.mark.parametrize("seed", range(6))
def test_random_rows_against_brute_force(seed):
    rng = np.random.default_rng(seed)
    for _ in range(40):
        V = int(rng.integers(1, 300))
        l = np.round(rng.normal(0, rng.choice([0.3, 2.0, 8.0]), V), int(rng.integers(0, 3))).astype(np.float32)
        l[rng.random(V) < rng.choice([0.0, 0.5, 0.95])] = -np.inf
        if not np.isfinite(l).any():
            l[int(rng.integers(V))] = 0.0
        T = float(rng.choice([0.6, 1.0, 2.0]))
        K = int(rng.choice([0, 1, 2, 20, 50, V - 1, V + 5]))
        P = float(rng.choice([1e-30, 0.5, 0.8, 0.9, 1.0]))
        check(l, T, max(K, 0), P)
