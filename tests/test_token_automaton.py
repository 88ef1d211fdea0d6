"""TokenAutomaton (calm_b200/lib.py), the host side of calm_b200_decode_sample_queue_constrained: the guided-choice trie,
next(), and every ValueError of the container (each one a case the C call would abort on).  No GPU needed."""
import numpy as np
import pytest

from calm_b200.lib import TokenAutomaton


def walk(a, seq, s=0):
    for t in seq:
        s = a.next(s, t)
    return s


def test_choices_trie():
    V = 100
    seqs = [[5, 7, 9], [5, 7, 3], [5, 8], [42], [5, 7, 9]]  # shared prefixes and a repeat
    a = TokenAutomaton.choices(seqs, V)
    # root, after 5, after 5 7, and one final state
    assert a.n_states == 4 and a.final.tolist() == [False, False, False, True]
    assert a.allowed(0).tolist() == [5, 42]
    assert a.allowed(walk(a, [5])).tolist() == [7, 8]
    assert a.allowed(walk(a, [5, 7])).tolist() == [3, 9]
    for q in seqs:
        assert a.final[walk(a, q)], q
        for j in range(len(q) - 1):  # no proper prefix ends
            assert not a.final[walk(a, q[:j + 1])]
    assert (a.next_default == -1).all()
    # every path from the root ends in exactly one of the choices
    ends, stack = set(), [(0, ())]
    while stack:
        s, p = stack.pop()
        if a.final[s]:
            ends.add(p)
            continue
        stack += [(a.next(s, int(t)), p + (int(t),)) for t in a.allowed(s)]
    assert ends == {tuple(q) for q in seqs}
    # the C layout: bitmask words, CSR exceptions ascending within a state
    assert a.allow.dtype == np.uint32 and a.allow.shape == (4, 4)
    assert a.exc_off.tolist() == [0, 2, 4, 6, 6]
    assert a.exc_tok.tolist() == [5, 42, 7, 8, 3, 9]


def test_choices_single_token_and_vocab_edge():
    V = 33  # a partial last word
    a = TokenAutomaton.choices([[32], [0]], V)
    assert a.allowed(0).tolist() == [0, 32] and a.allow[0].tolist() == [1, 1]
    assert a.final[a.next(0, 32)] and a.final[a.next(0, 0)]


def test_next_default_and_exceptions():
    V = 70
    allow = np.zeros((3, V), bool)
    allow[0, :] = True          # everything: loop unless 10 or 64
    allow[1, [3, 4]] = True
    a = TokenAutomaton(V, allow, [0, 0, -1], [{10: 1, 64: 2}, {3: 2}, None])
    assert a.next(0, 0) == 0 and a.next(0, 69) == 0 and a.next(0, 10) == 1 and a.next(0, 64) == 2
    assert a.next(1, 3) == 2 and a.next(1, 4) == 0
    assert a.final.tolist() == [False, False, True]
    assert a.allowed(1).tolist() == [3, 4] and len(a.allowed(0)) == V
    for s, t in ((1, 5), (2, 0), (0, V), (0, -1), (3, 0)):
        with pytest.raises(ValueError):
            a.next(s, t)
    # the bitmask form gives the same automaton
    b = TokenAutomaton(V, a.allow, a.next_default, [{10: 1, 64: 2}, {3: 2}, None])
    assert np.array_equal(a.allow, b.allow) and np.array_equal(a.exc_tok, b.exc_tok) and np.array_equal(a.exc_next, b.exc_next)


def test_container_errors():
    V = 40
    allow = np.zeros((2, V), bool)
    allow[0, [1, 2]] = True
    ok = dict(vocab=V, allow=allow, next_default=[1, -1], exceptions=[{2: 1}, None])
    TokenAutomaton(**ok)
    words = np.zeros((2, 2), np.uint32)
    words[0, 1] = 1 << (V % 32)  # token 40: past the vocabulary
    bad = [
        dict(vocab=0), dict(vocab=True),
        dict(allow=np.zeros(V, bool)),                 # not 2-D
        dict(allow=np.zeros((2, V + 1), bool)),        # a column per token
        dict(allow=np.zeros((2, 3), np.uint32)),       # wrong word count
        dict(allow=np.zeros((2, 2), np.int64)),        # wrong dtype
        dict(allow=words),                             # a bit past the vocabulary
        dict(next_default=[1]), dict(next_default=[1.0, -1.0]), dict(next_default=[2, -1]), dict(next_default=[-2, -1]),
        dict(next_default=[-1, -1]),                   # state 0 allows 1 outside its exceptions
        dict(exceptions=[{2: 1}]),                     # one per state
        dict(exceptions=[[2, 1], None]),               # not a dict
        dict(exceptions=[{3: 1}, None]),               # not allowed in its state
        dict(exceptions=[{V: 1}, None]), dict(exceptions=[{-1: 1}, None]), dict(exceptions=[{True: 1}, None]),
        dict(exceptions=[{2: 2}, None]), dict(exceptions=[{2: -1}, None]), dict(exceptions=[{2: 1.0}, None]),
    ]
    for b in bad:
        with pytest.raises(ValueError):
            TokenAutomaton(**{**ok, **b})
    for seqs in ([], [[]], [[1, 2], [1]], [[1], [1, 2]], [[V]], [[-1]]):
        with pytest.raises(ValueError):
            TokenAutomaton.choices(seqs, V)
