"""Binned inference on the H100: u8 tuples walked against the rank-coded layout (dte_load_ensemble_binned).

Bar everywhere: every score word and every label equals the oracle's on the fp32 tuples (or, on multi-device handles,
the engine's own fp32 path, which the rest of the suite holds to the oracle)."""
import numpy as np
import pytest

import ddt_b200 as ddt
from ddt_b200 import engine as E
from edge_operands import MISSING_ROTATION, edge_ensemble, edge_tuples, with_leaves
from helpers import (assert_scores, make_engine, multi_node_regs, oracle_scores, oracle_words, plan_groups, plan_rows,
                     refused, torch_cuda, write_regs, L)  # noqa: F401 (torch_cuda: a fixture)
from oracle import oracle as O

pytestmark = pytest.mark.gpu

VARIANTS = [E.DTE_KERNEL_GENERIC, E.DTE_KERNEL_TILE, E.DTE_KERNEL_TILE_STAGED, E.DTE_KERNEL_AUTO]


def matrix_cases():
    """One typical (|D - 10|, F smallest) and one extreme (largest D, F) row per (binned kernel template, C), as
    (row, None); then the typical row of every group on edge operands (tests/edge_operands.py), as (row, missing
    pattern) with the pattern taken from MISSING_ROTATION by group index."""
    out, edge = [], []
    for i, ((t, C), (typical, extreme)) in enumerate(plan_groups(plan_rows("plan_table_binned.txt.xz")).items()):
        for kind, r in (("typical", typical), ("extreme", extreme)):
            out.append(pytest.param(r, None, id="%s-C%d-%s-D%d-F%d" % (t.replace(" ", ""), C, kind, r.D, r.F)))
        m = MISSING_ROTATION[i % len(MISSING_ROTATION)]
        edge.append(pytest.param(typical, m, id="%s-C%d-edge-D%d-F%d-m%08x" % (t.replace(" ", ""), C, typical.D, typical.F, m)))
    return out + edge


def wave_tuples(name, sm_count=132):
    """Tuples of one wave of CTAs of a binned plan (32 x consumer warps / warps per group per CTA); 128 per block for
    the generic kernel."""
    if "tile" not in name:
        return 128 * sm_count
    pair = int(name.split("<")[1].split(",")[1])
    return sm_count * 32 * int(name.split("warps=")[1].split()[0]) // pair


def hist_ensemble(T, D, F, seed, cuts=254, wide=None):
    """L.synth_ensemble(cuts=); for F > 512 one node moves to feature F - 1 (wide records) with its threshold, so the
    cut count leaves room for that one extra edge."""
    if wide is None:
        wide = F > 512
    W, FI = L.synth_ensemble(T, D, F, seed=seed, cuts=cuts - 1 if wide else cuts)
    if wide:
        FI[0, (1 << D) - 2] = (FI[0, (1 << D) - 2] & 0x2000) | (F - 1)
    return W, FI


def run_case(torch, T, D, F, K, S, C, n, seed, variants=VARIANTS, missing=None):
    """Load binned; for every variant: host binned (bins from bin_edges + layout.bin_tuples) and device binned (bins from
    dte_bin_tuples_device on a non-default stream) against the oracle; the device bins equal the host bins byte for byte.
    missing given: edge operands (tests/edge_operands.py) with that missing pattern, the same trees loaded with wide and
    then with small leaves on one handle."""
    if missing is None:
        W, FI = hist_ensemble(T, D, F, seed)
        x = L.synth_tuples(0, n, F, seed=seed + 1, missing_ppm=20000)
        loads, missing = [W], L.MISSING_DEFAULT
    else:
        W, FI, pools = edge_ensemble(T, D, F, seed, leaves="wide", missing=missing)
        x = edge_tuples(n, F, pools, seed + 1, missing)
        loads = [W, with_leaves(W, D, "small", seed)]
    names = {}
    with make_engine(T, D, F, K, S, missing) as e:
        for Wl in loads:
            want = oracle_words(Wl, FI, x, D, K, S, C, missing)
            e.load_ensemble(*L.pack_streams(Wl, FI, D), num_classes=C, binned=True)
            off, edges = e.bin_edges()
            b = L.bin_tuples(x, off, edges, missing)
            dx = torch.from_numpy(x.view(np.int32)).cuda()
            db = torch.empty((n, F), dtype=torch.uint8, device="cuda")
            s = torch.cuda.Stream()
            e.bin_tuples_device(dx, n, db, stream=s.cuda_stream)
            s.synchronize()
            assert (db.cpu().numpy() == b).all(), "dte_bin_tuples_device differs from layout.bin_tuples"
            for v in variants:
                e.set_kernel_variant(v)
                names[v] = e.kernel_name_binned()
                sc, lb = e.infer_host_binned(b)
                assert_scores(sc, lb, want, C, "host %s" % names[v])
                ds = torch.empty((n, C) if C > 1 else (n,), dtype=torch.float32, device="cuda")
                dl = torch.empty(n, dtype=torch.uint8, device="cuda")
                e.infer_device_binned(db, n, ds, dl, stream=s.cuda_stream)
                s.synchronize()
                assert_scores(ds.cpu().numpy(), dl.cpu().numpy(), want, C, "device %s" % names[v])
            # the fp32 calls still score a binned load correctly
            e.set_kernel_variant(E.DTE_KERNEL_AUTO)
            sc, lb = e.infer_host(x)
            assert_scores(sc, lb, want, C, "fp32 after a binned load")
    return names


@pytest.mark.parametrize("row,missing", matrix_cases())
def test_reachable_binned_instantiation_bit_exact(torch_cuda, row, missing, monkeypatch):
    """Every binned kernel the planner reaches, with its pin, geometry and variant from the binned plan table; enough
    tuples for every CTA to walk two tiles.  Edge cases (missing given): edge operands on one wave of CTAs plus a ragged
    tail."""
    monkeypatch.setenv("DTE_TUNE", row.tune)
    T = 8 * 3 * max(1, row.C) if row.C > 1 else 40
    K, S = 1, 5
    if missing is None:
        n = 132 * 2 * 32 * 12 + 33 if row.variant != E.DTE_KERNEL_GENERIC else 5000
        n = min(n, 100_000 if row.F <= 512 else 20_000)
    else:
        n = wave_tuples(row.name) + 33
    names = run_case(torch_cuda, T, row.D, row.F, K, S, row.C, n, 1000 + row.D, variants=[row.variant], missing=missing)
    assert names[row.variant] == row.name


@pytest.mark.parametrize("D", [1, 2, 3, 4, 5, 12, 15])
def test_depths(torch_cuda, D):
    run_case(torch_cuda, 16 if D < 12 else 8, D, 256, 2, 4, 1, 3001, 2000 + D)


@pytest.mark.parametrize("F", [4, 12, 20, 256, 516, 2048])
def test_feature_counts(torch_cuda, F):
    run_case(torch_cuda, 24, 8, F, 4, 1, 1, 4099, 3000 + F)


def binned_tile(T, D, F, K, S):
    """Tuples per CTA of the binned plan the engine picks for this geometry (32 x consumer warps / warps per group)."""
    W, FI = hist_ensemble(T, D, F, 1)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F, K, S) as e:
        e.load_ensemble(wl, fl, binned=True)
        name = e.kernel_name_binned()
    pair = int(name.split("<")[1].split(",")[1])
    return 32 * int(name.split("warps=")[1].split()[0]) // pair


@pytest.mark.parametrize("which", ["1", "31", "33", "tile-1", "tile+1", "3-waves+7"])
def test_tuple_counts(torch_cuda, which):
    tile = binned_tile(24, 10, 128, 8, 1)
    n = {"1": 1, "31": 31, "33": 33, "tile-1": tile - 1, "tile+1": tile + 1, "3-waves+7": 132 * tile * 3 + 7}[which]
    run_case(torch_cuda, 24, 10, 128, 8, 1, 1, n, 4000 + n % 97)


@pytest.mark.parametrize("C,K,S", [(3, 2, 2), (256, 8, 1), (1, 1, 3), (1, 8, 1)])
def test_classes_and_slots(torch_cuda, C, K, S):
    T = 8 * C if C > 1 else 30
    run_case(torch_cuda, T, 6, 64, K, S, C, 2049, 5000 + C)


def test_phased_at_depth_5_stays_unphased(torch_cuda, monkeypatch):
    monkeypatch.setenv("DTE_TUNE", "pair=2,stages=1,phased=1")
    names = run_case(torch_cuda, 32, 5, 256, 2, 2, 1, 20_000, 6000, variants=[E.DTE_KERNEL_TILE_STAGED])
    assert " phased=0 " in names[E.DTE_KERNEL_TILE_STAGED]
    monkeypatch.setenv("DTE_TUNE", "pair=2,stages=1,phased=1")
    names = run_case(torch_cuda, 32, 6, 256, 2, 2, 1, 20_000, 6001, variants=[E.DTE_KERNEL_TILE_STAGED])
    assert " phased=1 " in names[E.DTE_KERNEL_TILE_STAGED]


def test_host_binned_on_multi_device_handles_and_pageable(torch_cuda):
    """Dealt and Chunked handles (two ring positions on one GPU), pinned and pageable bins: infer_host_binned equals
    infer_host on the fp32 tuples word for word; a line-stream-free fp32 call after it still works."""
    T, D, F, K, n = 40, 9, 128, 2, 70_001
    W, FI = hist_ensemble(T, D, F, 7000)
    x = L.synth_tuples(0, n, F, seed=7001, missing_ppm=15000)
    wl, fl = L.pack_streams(W, FI, D)
    for mode in ("data", "ensemble"):
        regs = multi_node_regs(T, D, F, K, n, 2, mode, batch_tuples=64)
        with ddt.Engine([0, 0]) as e:
            e.set_option(E.DTE_OPT_CHUNK_TUPLES, 5000)
            write_regs(e, regs)
            e.load_ensemble(wl, fl, binned=True)
            want, wlb = e.infer_host(x)
            off, edges = e.bin_edges()
            b = L.bin_tuples(x, off, edges)
            pinned = e.host_alloc(b.shape, np.uint8)
            pinned[:] = b
            for src in (b, pinned):
                sc, lb = e.infer_host_binned(src)
                assert (sc.view(np.uint32) == want.view(np.uint32)).all() and (lb == wlb).all(), mode
            e.host_free(pinned)
            sc, lb = e.infer_host(x)
            assert (sc.view(np.uint32) == want.view(np.uint32)).all(), mode
            refused(lambda: e.infer_device_binned(0, 0, 0), E.DTE_ERR_UNSUPPORTED)


def test_chunks_share_edges_and_ring_combine(torch_cuda):
    """Two single-device handles with different first_tree chunks export identical edges; their binned partials,
    ring-combined, equal the oracle's fp32 ring."""
    torch = torch_cuda
    T, D, F, K, S, n = 41, 8, 64, 2, 3, 3001
    W, FI = hist_ensemble(T, D, F, 7100)
    x = L.synth_tuples(0, n, F, seed=7101, missing_ppm=10000)
    wl, fl = L.pack_streams(W, FI, D)
    chunks = [(0, 20), (20, 21)]
    kw = dict(threads=O.max_threads())
    parts = [oracle_scores(W[a:a + c], FI[a:a + c], x, D, K, S, L.MISSING_DEFAULT, **kw) for a, c in chunks]
    want = O.ring_combine(parts)
    engines, bufs, tables = [], [], []
    for first, count in chunks:
        e = make_engine(T, D, F, K, S)
        e.load_ensemble(wl, fl, first_tree=first, num_local_trees=count, binned=True)
        tables.append(e.bin_edges())
        db = torch.from_numpy(L.bin_tuples(x, *tables[-1])).cuda()
        out = torch.empty(n, dtype=torch.float32, device="cuda")
        e.infer_device_binned(db, n, out)
        engines.append(e)
        bufs.append(out)
    assert (tables[0][0] == tables[1][0]).all() and (tables[0][1] == tables[1][1]).all()
    out = torch.empty(n, dtype=torch.float32, device="cuda")
    engines[0].ring_combine_device(bufs, n, out)
    assert (out.cpu().numpy().view(np.uint32) == want).all()
    for e in engines:
        e.close()


def test_refusals(torch_cuda):
    torch = torch_cuda
    T, D, F, K, S, n = 24, 6, 4, 1, 3, 1000                  # F = 4: ~380 live nodes per feature
    W, FI = hist_ensemble(T, D, F, 7200, cuts=20)
    x = L.synth_tuples(0, n, F, seed=7201)
    wl, fl = L.pack_streams(W, FI, D)
    want = oracle_words(W, FI, x, D, K, S, 1)
    with make_engine(T, D, F, K, S) as e:
        e.load_ensemble(wl, fl)
        refused(lambda: e.infer_host_binned(np.zeros((n, F), np.uint8)), E.DTE_ERR_STATE)      # binned call after a plain load
        refused(e.kernel_name_binned, E.DTE_ERR_STATE)
        d8 = torch.zeros(n * F, dtype=torch.uint8, device="cuda")
        d32 = torch.zeros(n * F, dtype=torch.float32, device="cuda")
        ds = torch.zeros(n, dtype=torch.float32, device="cuda")
        refused(lambda: e.infer_device_binned(d8, n, ds), E.DTE_ERR_STATE)
        refused(lambda: e.bin_tuples_device(d32, n, d8), E.DTE_ERR_STATE)
        Wb, FIb = L.synth_ensemble(T, D, F, seed=7202)       # U[0,1) thresholds: > 254 distinct on some feature
        wb, fb = L.pack_streams(Wb, FIb, D)
        refused(lambda: e.load_ensemble(wb, fb, binned=True), E.DTE_ERR_UNSUPPORTED, "distinct thresholds")
        sc, lb = e.infer_host(x)                              # the old ensemble still scores
        assert_scores(sc, lb, want, 1, "after a refused binned load")
        e.load_ensemble(wl, fl, binned=True)
        off = np.empty(F + 1, dtype=np.uint32)
        total = E.C.c_size_t()
        assert e._lib.dte_bin_edges(e._h, off.ctypes.data, None, 0, E.C.byref(total)) == 0 and total.value >= 2
        small = np.empty(total.value, dtype=np.uint32)
        assert e._lib.dte_bin_edges(e._h, off.ctypes.data, small.ctypes.data, total.value - 1, E.C.byref(total)) == E.DTE_ERR_ARG
        base = torch.zeros(n * F + 64, dtype=torch.uint8, device="cuda")
        scores = torch.zeros(n + 4, dtype=torch.float32, device="cuda")
        fx = torch.zeros(n * F + 16, dtype=torch.float32, device="cuda")
        for args in ((base.data_ptr() + 4, n, scores), (base.data_ptr(), n, scores.data_ptr() + 2)):
            refused(lambda: e.infer_device_binned(*args), E.DTE_ERR_ARG)
        refused(lambda: e.bin_tuples_device(fx.data_ptr() + 4, n, base), E.DTE_ERR_ARG)
        refused(lambda: e.bin_tuples_device(fx, n, base.data_ptr() + 8), E.DTE_ERR_ARG)
        e.load_ensemble(wl, fl)                               # a plain load drops the binned layout
        refused(e.bin_edges, E.DTE_ERR_STATE)


def test_headline_binned_multi_tile(torch_cuda):
    """cfg3-shaped hist ensemble (D = 12, F = 256) on the AUTO plan, several tiles per CTA; what tools/gpu_sanitize.sh
    runs for the binned walk."""
    names = run_case(torch_cuda, 64, 12, 256, 8, 1, 1, 132 * 320 * 2 + 5, 8000, variants=[E.DTE_KERNEL_AUTO])
    print("binned plan:", names[E.DTE_KERNEL_AUTO])
