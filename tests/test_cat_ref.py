"""The categorical restatement (tests/cat_ref.py) against hand-derived answers and against the oracle on the indicator
expansion (CPU only).

Bar: every KAT decision of tests/golden/categorical_kats.json as written; every score word of cat_ref.cat_scores equal
to the oracle's words on cat_ref.expand's ensemble, for random ensembles with D = 1..12, early leaves, C = 1 and 3 and
several K and S, so the two statements the GPU tests use as references agree with each other and with the edge cases."""
import json
import os

import numpy as np
import pytest

import ddt_b200 as ddt
from cat_ref import cat_scores, category, decide, expand, in_set, oracle_expanded

L = ddt.layout
HERE = os.path.dirname(os.path.abspath(__file__))


def kats():
    with open(os.path.join(HERE, "golden", "categorical_kats.json")) as fh:
        return json.load(fh)["cases"]


def set_words(spec):
    """A KAT set spec {len, members} -> its uint32 words."""
    w = np.zeros(spec["len"], dtype=np.uint64)
    for c in spec["members"]:
        w[c // 32] |= np.uint64(1) << np.uint64(c % 32)
    return w.astype(np.uint32)


def kat_node(case):
    """One D = 1 tree whose root is the KAT's categorical node (feature 0, set 0), leaves 1.0 left and 2.0 right."""
    words = set_words(case["set"])
    offsets = np.array([0, words.size], dtype=np.uint32)
    W = np.array([[0, 0x3F800000, 0x40000000]], dtype=np.uint32)
    FI = np.array([[0x8000 | (case["bit13"] << 13)]], dtype=np.uint16)
    return W, FI, offsets, words


@pytest.mark.parametrize("i", range(len(kats())))
def test_kat_decisions(i):
    c = kats()[i]
    words = set_words(c["set"])
    offsets = np.array([0, words.size], dtype=np.uint32)
    got = decide(int(c["x"], 16), 0, 0x8000 | (c["bit13"] << 13), int(c["missing"], 16), offsets, words)
    assert got == bool(c["right"]), c["why"]


def test_kat_words_through_the_expansion():
    """Every KAT as a one-node tree: the restatement's score and the oracle's on the expansion are the leaf of the
    KAT's direction."""
    for c in kats():
        if c["set"]["len"] > 4:
            continue                                   # the 2^19-word set is covered by test_kat_decisions
        W, FI, offsets, words = kat_node(c)
        x = np.array([[int(c["x"], 16), 0, 0, 0]], dtype=np.uint32)
        m = int(c["missing"], 16)
        want = 0x40000000 if c["right"] else 0x3F800000
        assert cat_scores(W, FI, x, 1, 1, 1, m, offsets, words)[0] == want, c["why"]
        assert oracle_expanded(W, FI, x, 1, 1, 1, m, offsets, words)[0] == want, c["why"]


def test_category_rule():
    assert category(0x80000000) == 0 and category(0x00000000) == 0 and category(0x00000001) == 0
    assert category(0x4B7FFFFF) == (1 << 24) - 1 and category(0x4B800000) is None
    assert category(0xBF000000) is None and category(0x7FC00000) is None and category(0x402CCCCD) == 2
    assert in_set(32, np.array([0, 1], np.uint32)) and not in_set(64, np.array([0, 1], np.uint32))


def early(FI, D, rng, p=0.15):
    """Bit 14 on a random share of internal nodes above the last level."""
    FI = FI.copy()
    n_up = (1 << (D - 1)) - 1
    if n_up:
        FI[:, :n_up] |= (rng.random((FI.shape[0], n_up)) < p).astype(np.uint16) << np.uint16(14)
    return FI


def random_case(D, T, F, seed, share, n, C_f=(3, 40, 100)):
    rng = np.random.default_rng(seed)
    W, FI = L.synth_ensemble(T, D, F, seed=seed)
    FI = early(FI, D, rng) if D >= 3 else FI
    cat_f = rng.choice(F, size=min(3, F), replace=False)
    C_f = np.array(C_f[:cat_f.size])
    W, FI, offsets, words = L.synth_categorical(W, FI, D, cat_f, C_f, share=share, seed=seed + 1)
    x = L.synth_tuples(seed, n, F, missing_ppm=50000)
    x = L.categorical_tuples(x, cat_f, C_f + 8, seed=seed + 2)      # some codes past each set's categories
    # edge words in the categorical columns: invalid values, -0, fractions, the missing pattern
    edge = np.array([0x80000000, 0x3F000000, 0x402CCCCD, 0x7FC00000, 0xBF800000, 0x7F800000, 0x4B800000, 0x00000001],
                    dtype=np.uint32)
    for f in cat_f:
        hit = rng.random(n) < 0.2
        x[hit, f] = rng.choice(edge, size=int(hit.sum()))
    return W, FI, offsets, words, x


CASES = [(1, 16, 4, 1, 1, 1), (2, 16, 8, 2, 1, 1), (3, 24, 8, 8, 1, 1), (4, 40, 16, 2, 3, 1), (5, 16, 8, 1, 2, 1),
         (6, 24, 12, 4, 1, 1), (8, 16, 20, 8, 1, 1), (10, 8, 16, 1, 8, 1), (12, 4, 32, 2, 2, 1),
         (1, 27, 8, 1, 4, 3), (3, 30, 8, 2, 2, 3), (5, 33, 12, 8, 1, 3), (7, 24, 16, 1, 3, 3), (9, 12, 8, 4, 1, 3),
         (12, 6, 16, 1, 1, 3)]


@pytest.mark.parametrize("D,T,F,K,S,C", CASES)
def test_restatement_equals_oracle_on_expansion(D, T, F, K, S, C):
    share = 0.5 if D <= 6 else 0.1 if D <= 9 else 0.02
    W, FI, offsets, words, x = random_case(D, T, F, 1000 + 17 * D + T, share, 48)
    assert (FI & 0x8000).any()
    for missing in (L.MISSING_DEFAULT, 0x00000000):
        if C >= 2 and 8 * S * K < -(-T // C):
            S = -(-(-(-T // C)) // (8 * K))
        got = cat_scores(W, FI, x, D, K, S, missing, offsets, words, C=C)
        want = oracle_expanded(W, FI, x, D, K, S, missing, offsets, words, C=C)
        assert (got == want).all(), (D, T, F, K, S, C, hex(missing), int((got != want).sum()))


def test_dead_categorical_bits_are_ignored():
    """Bit 15 below an early leaf changes nothing: its weight word may be any set number."""
    D, F = 3, 4
    W = np.array([[0, 0x3F000000, 0x3F000000, 7, 99, 5, 0xFFFFFFFF, 1, 2, 3, 4, 5, 6, 7, 8]], dtype=np.uint32)
    W[0, 7:] = np.arange(1, 9, dtype=np.float32).view(np.uint32)
    FI = np.array([[0x8000, 0x4001, 0x0002, 0x8000, 0x8001, 0x0003, 0x0002]], dtype=np.uint16)
    offsets, words = np.array([0, 1], np.uint32), np.array([0xFFFFFFFF], np.uint32)
    x = L.synth_tuples(3, 64, F)
    want = oracle_expanded(W, FI, x, D, 1, 1, L.MISSING_DEFAULT, offsets, words)
    assert (cat_scores(W, FI, x, D, 1, 1, L.MISSING_DEFAULT, offsets, words) == want).all()
    W2, FI2, _ = expand(W, FI, x, D, L.MISSING_DEFAULT, offsets, words)
    assert FI2[0, 0] == 4 and (FI2[0, 1:] == FI[0, 1:] & 0x7FFF).all()   # only the root got a column; 3 and 4 are dead


def test_generator_shapes():
    W, FI = L.synth_ensemble(8, 6, 16)
    W2, FI2, off, words = L.synth_categorical(W, FI, 6, [1, 5], [4, 1000], share=0.3, seed=5)
    cat = (FI2 & 0x8000) != 0
    assert cat.any() and (np.diff(off.astype(np.int64)) > 0).all() and off[-1] == words.size
    assert set(np.unique(FI2[cat] & 0x7FF)) <= {1, 5}
    n_int = FI.shape[1]
    assert (W2[:, :n_int][cat] < off.size - 1).all() and (W2[:, :n_int][~cat] == W[:, :n_int][~cat]).all()
    assert (W2[:, n_int:] == W[:, n_int:]).all()
    for s in range(off.size - 1):
        n_words = off[s + 1] - off[s]
        assert n_words in (1, 32)
        if n_words == 1:
            assert words[off[s]] < 16                  # 4 categories: bits 0..3 only
        else:
            assert words[off[s + 1] - 1] < (1 << 8)    # 1000 = 31 * 32 + 8 categories
    x = L.categorical_tuples(L.synth_tuples(0, 100, 16), [1, 5], [4, 1000])
    c1 = x[:, 1][x[:, 1] != L.MISSING_DEFAULT].view(np.float32)
    assert c1.min() >= 0 and c1.max() <= 3 and (c1 == np.floor(c1)).all()
