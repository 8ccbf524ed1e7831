"""Categorical splits on the H100 (dte_load_ensemble_categorical, dte_infer_*_categorical; DESIGN.md §16).

Bar everywhere: every score word and label equals the oracle's on the indicator expansion (tests/cat_ref.oracle_expanded;
the restatement cat_ref.cat_scores where the expansion would pass 2^11 feature indices), for dt_walk_tile_cat and the
forced dt_walk_generic_cat, on the device and through the host landing pipeline."""
import json
import os

import numpy as np
import pytest

import ddt_b200 as ddt
from ddt_b200 import engine as E
from cat_ref import cat_scores, oracle_expanded
from edge_operands import MISSING_ROTATION, edge_ensemble, edge_tuples, with_early_leaves
from helpers import (assert_scores, device_scores, geometry_regs, labels_of, make_engine, multi_node_regs,
                     oracle_scores, refused, torch_cuda, write_regs, L)  # noqa: F401 (torch_cuda: a fixture)

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def categorical_case(T, D, F, seed, share, n, C_f=(5, 40, 300), early=False, cat_f=None):
    rng = np.random.default_rng(seed)
    W, FI = L.synth_ensemble(T, D, F, seed=seed)
    if early and D >= 2:
        W, FI = with_early_leaves(W, FI, D, seed, leaves="small", per_tree=1)
    cat_f = np.asarray(cat_f if cat_f is not None else rng.choice(F, size=min(3, F), replace=False))
    C_f = np.resize(np.asarray(C_f), cat_f.size)
    W, FI, off, words = L.synth_categorical(W, FI, D, cat_f, C_f, share=share, seed=seed + 1)
    x = L.synth_tuples(seed, n, F, missing_ppm=30000)
    x = L.categorical_tuples(x, cat_f, C_f + 8, seed=seed + 2)
    return W, FI, off, words, x


def reference(W, FI, x, D, K, S, missing, off, words, C=1):
    n_cat = int(((FI & 0x8000) != 0).sum())
    if x.shape[1] + n_cat <= 2048:
        return oracle_expanded(W, FI, x, D, K, S, missing, off, words, C=C)
    return cat_scores(W, FI, x, D, K, S, missing, off, words, C=C)


def check(torch, e, x, want, C, variants=(E.DTE_KERNEL_TILE, E.DTE_KERNEL_GENERIC), what=""):
    names = []
    for v in variants:
        e.set_kernel_variant(v)
        name = e.kernel_name_categorical()
        names.append(name)
        if v == E.DTE_KERNEL_GENERIC:
            assert name.startswith("dt_walk_generic_cat"), name
        sc, lb = e.infer_host_categorical(x)
        assert_scores(sc, lb, want, C, "%s host %s" % (what, name))
        s = torch.cuda.Stream()
        dsc, dlb = device_scores(torch, e, "_categorical", x, C, stream=s.cuda_stream)
        assert_scores(dsc, dlb, want, C, "%s device %s" % (what, name))
    e.set_kernel_variant(E.DTE_KERNEL_AUTO)
    return names


# (D, T, F, K, S, C, n): D = 1..15, one and three classes, n across warp and tile edges and several waves
CASES = [(1, 16, 8, 1, 1, 1, 33), (2, 24, 16, 2, 1, 1, 31), (3, 20, 8, 8, 1, 1, 32), (4, 40, 16, 1, 3, 1, 1),
         (5, 64, 64, 8, 1, 1, 1000), (6, 32, 16, 2, 2, 1, 120000), (7, 48, 32, 4, 1, 1, 385), (8, 64, 128, 2, 2, 1, 4097),
         (9, 16, 64, 1, 2, 1, 700), (10, 32, 256, 4, 1, 1, 3000), (11, 8, 64, 1, 1, 1, 400), (12, 16, 64, 1, 2, 1, 700),
         (13, 8, 32, 1, 1, 1, 300), (14, 8, 16, 2, 1, 1, 129), (15, 8, 16, 1, 1, 1, 200),
         (1, 27, 8, 1, 4, 3, 129), (3, 30, 8, 2, 2, 3, 33), (5, 33, 32, 8, 1, 3, 2000), (7, 33, 32, 2, 2, 3, 500),
         (9, 12, 16, 1, 1, 3, 300), (11, 12, 64, 1, 1, 3, 300), (13, 9, 16, 1, 1, 3, 100), (15, 6, 8, 1, 1, 3, 64)]


@pytest.mark.parametrize("D,T,F,K,S,C,n", CASES)
def test_bit_exact_against_the_expansion(torch_cuda, D, T, F, K, S, C, n):
    share = min(0.5, 400.0 / (T * ((1 << D) - 1)))     # about 400 categorical nodes at most: the expansion stays narrow
    W, FI, off, words, x = categorical_case(T, D, F, 4000 + 31 * D + T + C, share, n, early=D >= 3)
    if C >= 2:
        S = max(S, -(-(-(-T // C)) // (8 * K)))
    want = reference(W, FI, x, D, K, S, L.MISSING_DEFAULT, off, words, C=C)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F, K, S) as e:
        e.load_ensemble(wl, fl, num_classes=C, categories=(off, words))
        names = check(torch_cuda, e, x, want, C, what="D=%d C=%d" % (D, C))
        assert names[0].startswith("dt_walk_tile_cat<"), names
        if C >= 2:
            assert names[0].endswith(" classes=%d" % C)
        e.infer_host_categorical(x[:0])                  # n = 0 is a no-op
        e.infer_device_categorical(0, 0, 0)


@pytest.mark.parametrize("F", [1816, 1820, 2048])
def test_tile_generic_boundary_and_widest_tuples(torch_cuda, F):
    """F = 1816 is the widest tuple group the tile holds in the H100's 227 KiB; from 1820 every variant runs the generic
    walk; F = 2048 reaches feature index 2047 on a categorical node."""
    T, D, K, n = 16, 6, 2, 300
    W, FI, off, words, x = categorical_case(T, D, F, 77 + F, 0.3, n, cat_f=[F - 1, 3, F // 2])
    want = reference(W, FI, x, D, K, 1, L.MISSING_DEFAULT, off, words)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F, K, 1) as e:
        e.load_ensemble(wl, fl, categories=(off, words))
        names = check(torch_cuda, e, x, want, 1, variants=(E.DTE_KERNEL_TILE, E.DTE_KERNEL_TILE_STAGED, E.DTE_KERNEL_GENERIC))
        fits = F * 128 <= 232448
        assert names[0].startswith("dt_walk_tile_cat<4> warps=1" if fits else "dt_walk_generic_cat"), names


@pytest.mark.parametrize("missing", MISSING_ROTATION)
def test_edge_operands_in_every_feature(torch_cuda, missing):
    """Edge words in every feature (tests/edge_operands.py) on numeric and categorical nodes alike, with early leaves."""
    T, D, F, K, n = 32, 6, 16, 4, 2000
    W, FI, pools = edge_ensemble(T, D, F, seed=missing & 0xFFFF, leaves="wide", missing=missing)
    W, FI = with_early_leaves(W, FI, D, seed=5, leaves="wide", root_trees=(3,))
    W, FI, off, words = L.synth_categorical(W, FI, D, np.arange(F), [2, 33, 64, 100] * (F // 4), share=0.4, seed=missing & 0xFFF)
    x = edge_tuples(n, F, pools, seed=9, missing=missing)
    codes = L.categorical_tuples(x, np.arange(F), 110, seed=11, missing=missing)
    x = np.where(np.random.default_rng(13).random(x.shape) < 0.4, codes, x).astype(np.uint32)
    want = reference(W, FI, x, D, K, 1, missing, off, words)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F, K, 1, missing=missing) as e:
        e.load_ensemble(wl, fl, categories=(off, words))
        check(torch_cuda, e, x, want, 1, what="missing 0x%08X" % missing)


def test_kats_on_the_device(torch_cuda):
    """Every hand-derived decision of tests/golden/categorical_kats.json: tree k of a group is the KAT's node on feature
    k, leaves +0 left and 2^k right, so the score's bits are the directions."""
    with open(os.path.join(HERE, "golden", "categorical_kats.json")) as fh:
        cases = json.load(fh)["cases"]
    by_missing = {}
    for c in cases:
        by_missing.setdefault(c["missing"], []).append(c)
    groups = [(m, g[i:i + 20]) for m, g in by_missing.items() for i in range(0, len(g), 20)]   # sums below 2^20: exact
    for m, group in groups:
        T = len(group)
        F = -(-T // 4) * 4
        W = np.zeros((T, 3), dtype=np.uint32)
        FI = np.zeros((T, 1), dtype=np.uint16)
        offsets, words = [0], []
        x = np.zeros((1, F), dtype=np.uint32)
        for k, c in enumerate(group):
            w = np.zeros(c["set"]["len"], dtype=np.uint64)
            for cat in c["set"]["members"]:
                w[cat // 32] |= np.uint64(1) << np.uint64(cat % 32)
            words += list(w.astype(np.uint32))
            offsets.append(len(words))
            W[k] = [k, 0, np.float32(2.0 ** k).view(np.uint32)]
            FI[k, 0] = 0x8000 | (c["bit13"] << 13) | k
            x[0, k] = int(c["x"], 16)
        off, words = np.array(offsets, np.uint32), np.array(words, np.uint32)
        wl, fl = L.pack_streams(W, FI, 1)
        with make_engine(T, 1, F, 1, -(-T // 8), missing=int(m, 16)) as e:
            e.load_ensemble(wl, fl, categories=(off, words))
            for v in (E.DTE_KERNEL_TILE, E.DTE_KERNEL_GENERIC):
                e.set_kernel_variant(v)
                bits = int(e.infer_host_categorical(x)[0][0])
                dsc, _ = device_scores(torch_cuda, e, "_categorical", x, 1)
                assert dsc[0] == np.float32(bits).view(np.uint32)
                for k, c in enumerate(group):
                    assert (bits >> k) & 1 == c["right"], (c["why"], E.KERNEL_NAMES[v])


def test_missing_pattern_rewritten_after_the_load(torch_cuda):
    T, D, F, K, n = 24, 5, 16, 2, 1500
    W, FI, off, words, x = categorical_case(T, D, F, 611, 0.5, n)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F, K, 2) as e:
        e.load_ensemble(wl, fl, categories=(off, words))
        for missing in (0x40000000, 0x00000000, L.MISSING_DEFAULT):   # 2.0 and +0 are valid category words
            x2 = x.copy()
            x2[::7, 1] = missing
            x2[::5, 2] = missing
            write_regs(e, {205: geometry_regs(T, D, F, K, 2, missing)[205]})
            check(torch_cuda, e, x2, reference(W, FI, x2, D, K, 2, missing, off, words), 1, what="missing 0x%08X" % missing)


@pytest.mark.parametrize("D,T,F,C", [(1, 16, 8, 1), (6, 64, 64, 1), (10, 32, 256, 1), (7, 33, 32, 3)])
def test_no_sets_is_the_fp32_walk(torch_cuda, D, T, F, C):
    """n_sets = 0: the categorical walk's words are dte_infer_device's on a plain load of the same streams."""
    K, n = 4, 5000
    W, FI = L.synth_ensemble(T, D, F, seed=D * 7 + T)
    x = L.synth_tuples(1, n, F)
    wl, fl = L.pack_streams(W, FI, D)
    S = max(1, -(-(-(-T // C)) // (8 * K)))
    with make_engine(T, D, F, K, S) as e:
        e.load_ensemble(wl, fl, num_classes=C)
        dx = torch_cuda.from_numpy(x.view(np.int32)).cuda()
        ds = torch_cuda.empty(n * C, dtype=torch_cuda.float32, device="cuda")
        e.infer_device(dx, n, ds)
        want = ds.cpu().numpy().view(np.uint32)
        want = want if C == 1 else want.reshape(n, C)
        for cats in ((None, None), (np.zeros(1, np.uint32), np.zeros(0, np.uint32))):
            e.load_ensemble(wl, fl, num_classes=C, categories=cats)
            check(torch_cuda, e, x, want, C, what="no sets")
    if C == 1:
        assert (want == oracle_scores(W, FI, x, D, K, S, L.MISSING_DEFAULT)).all()


def test_host_path_pinned_and_pageable(torch_cuda):
    T, D, F, K, n = 48, 8, 64, 4, 70001
    W, FI, off, words, x = categorical_case(T, D, F, 8080, 0.2, n)
    want = reference(W, FI, x, D, K, 2, L.MISSING_DEFAULT, off, words)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F, K, 2) as e:
        e.set_option(E.DTE_OPT_CHUNK_TUPLES, 9000)
        e.load_ensemble(wl, fl, categories=(off, words))
        hx = e.host_alloc(x.shape, np.uint32)
        hs = e.host_alloc((n,), np.float32)
        hx[:] = x
        sc, lb = e.infer_host_categorical(hx, out_scores=hs)
        assert (hs.view(np.uint32) == want).all() and (lb == labels_of(want, 1)).all()
        sc, lb = e.infer_host_categorical(x)
        assert (sc.view(np.uint32) == want).all()
        e.host_free(hx)
        e.host_free(hs)


@pytest.mark.parametrize("mode", ["data", "ensemble"])
def test_dealt_and_chunked_handles(mode):
    """Three ring positions sharing GPU 0: Dealt rows in global order, Chunked partials ring-combined in ring order."""
    G, T, D, F, K, n = 3, 48, 6, 32, 2, 4001
    W, FI, off, words, x = categorical_case(T, D, F, 3131, 0.4, n)
    S = -(-(-(-T // G)) // (8 * K)) if mode == "ensemble" else -(-T // (8 * K))
    if mode == "data":
        want = reference(W, FI, x, D, K, S, L.MISSING_DEFAULT, off, words)
    else:
        from oracle import oracle as O
        parts = []
        for g in range(G):
            first, count = ddt.sharding.ensemble_chunk(T, g, G)
            parts.append(reference(W[first:first + count], FI[first:first + count], x, D, K, S, L.MISSING_DEFAULT, off, words))
        want = O.ring_combine(parts)
    wl, fl = L.pack_streams(W, FI, D)
    with ddt.Engine([0, 0, 0]) as e:
        e.set_option(E.DTE_OPT_CHUNK_TUPLES, 700)
        write_regs(e, multi_node_regs(T, D, F, K, n, G, mode, batch_tuples=64))
        e.load_ensemble(wl, fl, categories=(off, words))
        for v in (E.DTE_KERNEL_TILE, E.DTE_KERNEL_GENERIC):
            e.set_kernel_variant(v)
            sc, lb = e.infer_host_categorical(x)
            assert (sc.view(np.uint32) == want).all(), (mode, E.KERNEL_NAMES[v])
            assert (lb == labels_of(want, 1)).all()
        refused(lambda: e.infer_device_categorical(0x1000, 4, 0x2000), E.DTE_ERR_UNSUPPORTED)   # device pointers belong to one device


def test_refusals(torch_cuda):
    T, D, F, K, n = 16, 4, 8, 2, 64
    W, FI, off, words, x = categorical_case(T, D, F, 9090, 0.5, n)
    want = reference(W, FI, x, D, K, 1, L.MISSING_DEFAULT, off, words)
    wl, fl = L.pack_streams(W, FI, D)
    dx = torch_cuda.from_numpy(x.view(np.int32)).cuda()
    ds = torch_cuda.empty(n + 4, dtype=torch_cuda.float32, device="cuda")
    cov = L.synth_covers(FI & 0x7FFF, D)
    with make_engine(T, D, F, K, 1) as e:
        # before any categorical load: the categorical calls name their load
        e.load_ensemble(wl, fl)
        plain = e.infer_host(x)[0].copy()
        for call in (lambda: e.infer_host_categorical(x), lambda: e.infer_device_categorical(dx, n, ds),
                     lambda: e.kernel_name_categorical()):
            refused(call, E.DTE_ERR_STATE, "no categorical layout resident: load the ensemble with dte_load_ensemble_categorical")
        for kw in (dict(binned=True), dict(covers=cov), dict(covers=cov, approx=True), dict(background=x[:4])):
            with pytest.raises(ValueError):
                e.load_ensemble(wl, fl, categories=(off, words), **kw)
        # refused loads leave the previous ensemble answering
        tc, nc = np.nonzero(FI & 0x8000)
        t0, node = int(tc[0]), int(nc[0])                # the first categorical node, set 0
        last = off.size - 2                              # the last one holds the last set, which a shorter CSR lacks
        refused(lambda: e.load_ensemble(wl, fl, categories=(off[:-1], words)), E.DTE_ERR_ARG,
                "tree %d node %d: categorical node with set number %d, but %d sets were given" % (tc[-1], nc[-1], last, last))
        bad = off.copy()
        bad[2] = bad[3] + 1
        refused(lambda: e.load_ensemble(wl, fl, categories=(bad, words)), E.DTE_ERR_ARG,
                "dte_load_ensemble_categorical: set_offsets decreases at set 2")
        big = np.array([0, (1 << 19) + 1], np.uint32)
        refused(lambda: e.load_ensemble(wl, fl, categories=(big, np.zeros((1 << 19) + 1, np.uint32))), E.DTE_ERR_UNSUPPORTED,
                "dte_load_ensemble_categorical: set 0 has 524289 words: a set holds at most 2^19 words")
        FIw = FI.copy()
        FIw[t0, node] = (FIw[t0, node] & ~np.uint16(0x7FF)) | np.uint16(F)
        refused(lambda: e.load_ensemble(*L.pack_streams(W, FIw, D), categories=(off, words)), E.DTE_ERR_UNSUPPORTED,
                "tree %d node %d: feature index %d >= %d features" % (t0, node, F, F))
        assert (e.infer_host(x)[0].view(np.uint32) == plain.view(np.uint32)).all()
        # a categorical load: every other kind is refused with a message naming the categorical calls
        e.load_ensemble(wl, fl, categories=(off, words))
        assert (e.infer_host_categorical(x)[0].view(np.uint32) == want).all()
        acc = torch_cuda.zeros(n, dtype=torch_cuda.float32, device="cuda")
        others = [lambda: e.infer_host(x), lambda: e.infer_device(dx, n, ds), lambda: e.infer_device_accumulate(dx, n, acc),
                  lambda: e.infer_host_sparse((np.zeros(n + 1, np.int64), np.zeros(0, np.uint32), np.zeros(0, np.uint32))),
                  lambda: e.infer_host_binned(np.zeros((n, F), np.uint8)), lambda: e.infer_host_leaves(x),
                  lambda: e.infer_host_contribs(x), lambda: e.infer_host_approx_contribs(x),
                  lambda: e.infer_host_interventional(x), lambda: e.infer_host_interactions(x),
                  lambda: e.infer_device_leaves(dx, n, ds), lambda: e.kernel_name(), lambda: e.kernel_name_leaves(),
                  lambda: e.kernel_name_contribs()]
        for call in others:
            refused(call, E.DTE_ERR_STATE, "a categorical ensemble is resident: walk it with dte_infer_device_categorical / "
                                           "dte_infer_host_categorical")
        refused(lambda: e.autotune(1000), E.DTE_ERR_STATE, "dte_autotune times the fp32 walk's plans")
        # misaligned pointers are refused before any launch
        raw = torch_cuda.empty(n * F + 8, dtype=torch_cuda.int32, device="cuda")
        refused(lambda: e.infer_device_categorical(raw.data_ptr() + 4, n, ds), E.DTE_ERR_ARG,
                "dte_infer_device_categorical: d_tuples not 16-byte aligned")
        refused(lambda: e.infer_device_categorical(dx, n, ds.data_ptr() + 2), E.DTE_ERR_ARG,
                "dte_infer_device_categorical: d_scores not 4-byte aligned")
        # a tuple-only line stream cannot reuse a categorical ensemble
        regs = geometry_regs(T, D, F, K, 1, L.MISSING_DEFAULT, n)
        regs[201] = (regs[201] & ~0x2) | 0x1 | 0x40              # data_distributed, no host node: the run reuses the ensemble
        write_regs(e, regs)
        refused(lambda: e.start(), E.DTE_ERR_CONFIG, "a categorical ensemble is resident: the line stream walks numeric trees only")
        write_regs(e, geometry_regs(T, D, F, K, 1, L.MISSING_DEFAULT))
        assert (e.infer_host_categorical(x)[0].view(np.uint32) == want).all()
        # any other placement drops the categorical layout
        e.load_ensemble(wl, fl, covers=cov)
        refused(lambda: e.infer_host_categorical(x), E.DTE_ERR_STATE, "dte_load_ensemble_categorical")
        e.load_ensemble(wl, fl, leaves=True)
        refused(lambda: e.kernel_name_categorical(), E.DTE_ERR_STATE, "dte_load_ensemble_categorical")
        assert (e.infer_host(x)[0].view(np.uint32) == plain.view(np.uint32)).all()
        info = e.info()
        e.load_ensemble(wl, fl, categories=(off, words), leaves=True)   # no leaf layout next to a categorical one
        refused(lambda: e.infer_host_leaves(x), E.DTE_ERR_STATE, "a categorical ensemble is resident")
        assert e.info()["ensemble_bytes"] > 0 and e.info()["num_classes"] == 1 and info["num_classes"] == 1
