"""Leaf-index inference on the H100 (dte_infer_device_leaves / dte_infer_host_leaves).

Bar everywhere: every cell equals the oracle's (tests/leaf_oracle.py: the oracle's own walk over trees whose end
cells are labelled with their index), and the scores rebuilt from the cells with the oracle's adder equal the same
handle's score words."""
import numpy as np
import pytest

import ddt_b200 as ddt
from ddt_b200 import engine as E
from edge_operands import MISSING_ROTATION, edge_ensemble, edge_tuples
from helpers import (assert_words, early, make_engine, multi_node_regs, plan_groups, plan_rows, refused, torch_cuda,
                     write_regs, L)  # noqa: F401 (torch_cuda: a fixture)
from leaf_oracle import leaf_cells
from oracle import oracle as O

pytestmark = pytest.mark.gpu

VARIANTS = [E.DTE_KERNEL_GENERIC, E.DTE_KERNEL_TILE, E.DTE_KERNEL_TILE_STAGED, E.DTE_KERNEL_AUTO]


def device_leaves(torch, e, x, T, stream=None, offset=0):
    n = x.shape[0]
    dx = torch.from_numpy(x.view(np.int32)).cuda()
    buf = torch.full((offset + n * T + 8,), 0x7777, dtype=torch.int16, device="cuda")
    out = buf[offset: offset + n * T]
    e.infer_device_leaves(dx, n, out, stream=stream)
    torch.cuda.synchronize()
    assert (buf[offset + n * T:].cpu().numpy() == 0x7777).all(), "wrote past the last row"
    return out.cpu().numpy().view(np.uint16).reshape(n, T)


def run(torch, T, D, F, n, seed, C=1, variants=VARIANTS, early_leaves=True, K=8, S=None):
    W, FI = L.synth_ensemble(T, D, F, seed=seed)
    if early_leaves and D >= 2:
        FI = early(FI, D, seed)
    x = L.synth_tuples(0, n, F, seed=seed + 1, missing_ppm=20000)
    wl, fl = L.pack_streams(W, FI, D)
    want = leaf_cells(W, FI, x, D, L.MISSING_DEFAULT)
    with make_engine(T, D, F, K, S) as e:
        e.load_ensemble(wl, fl, num_classes=C, leaves=True)
        for v in variants:
            e.set_kernel_variant(v)
            assert_words(e.infer_host_leaves(x), want, "host %s" % E.KERNEL_NAMES[v])
            s = torch.cuda.Stream()
            assert_words(device_leaves(torch, e, x, T, stream=s.cuda_stream), want, "device %s" % E.KERNEL_NAMES[v])
    return W, FI, x, want


def matrix_cases():
    """(row, whole, missing): one typical and one extreme row per (leaf kernel template, C) of the leaf plan table, each
    at a ragged and at a whole T on the standard data (missing None); then the typical row of every group at the ragged
    T on edge operands (tests/edge_operands.py), the missing pattern taken from MISSING_ROTATION by group index."""
    out, edge = [], []
    for i, ((t, C), (typical, extreme)) in enumerate(plan_groups(plan_rows("plan_table_leaf.txt.xz")).items()):
        for kind, r in (("typical", typical), ("extreme", extreme)):
            for whole, wid in ((False, "T-ragged"), (True, "T-whole")):
                out.append(pytest.param(r, whole, None, id="%s-C%d-%s-D%d-F%d-%s" % (t.replace(" ", ""), C, kind, r.D, r.F, wid)))
        m = MISSING_ROTATION[i % len(MISSING_ROTATION)]
        edge.append(pytest.param(typical, False, m, id="%s-C%d-edge-D%d-F%d-m%08x-T-ragged" % (
            t.replace(" ", ""), C, typical.D, typical.F, m)))
    return out + edge


@pytest.mark.parametrize("row,whole,missing", matrix_cases())
def test_every_reachable_leaf_kernel(torch_cuda, row, whole, missing, monkeypatch):
    """Pin the row's DTE_TUNE and variant, check the kernel name, and walk two tiles per CTA.  T-ragged: T not a
    multiple of 8 (one class: the 2-byte cell stores; several: padding slots).  T-whole: T = 32 per class, so a
    one-class walk takes the 2*ILP-byte vector stores.  Edge cases (missing given): edge operands with early leaves
    and that missing pattern on one wave of CTAs plus a ragged tail."""
    monkeypatch.setenv("DTE_TUNE", row.tune)
    D, F, C = row.D, row.F, row.C
    T = 32 * C if whole else 32 * C - (3 if C > 1 else 5)
    edge = missing is not None
    if not edge:
        W, FI = L.synth_ensemble(T, D, F, seed=800 + D)
        if F > 512:
            FI[0, (1 << D) - 2] = (FI[0, (1 << D) - 2] & 0x2000) | (F - 1)
        missing = L.MISSING_DEFAULT
    else:
        W, FI, pools = edge_ensemble(T, D, F, seed=850 + D, missing=missing)
    if D >= 2:
        FI = early(FI, D, D)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F, missing=missing) as e:
        e.load_ensemble(wl, fl, num_classes=C, leaves=True)
        e.set_kernel_variant(row.variant)
        name = e.kernel_name_leaves()
        assert name == row.name, (name, row.name)
        tpc = int(e.info()["tuples_per_cta"]) if "tile" in name else 128
        if edge:
            n = 132 * tpc + 7
            x = edge_tuples(n, F, pools, seed=851 + D, missing=missing)
        else:
            n = min(2 * 132 * tpc + 7, max(4096, 300000 // max(1, F)))
            x = L.synth_tuples(0, n, F, seed=801, missing_ppm=20000)
        want = leaf_cells(W, FI, x, D, missing)
        s = torch_cuda.cuda.Stream()
        assert_words(device_leaves(torch_cuda, e, x, T, stream=s.cuda_stream), want, name)


@pytest.mark.parametrize("D", list(range(1, 16)))
def test_depths(torch_cuda, D):
    run(torch_cuda, 19 if D < 14 else 9, D, 32, 700, 900 + D)


@pytest.mark.parametrize("n", [0, 1, 31, 33])
def test_small_batches(torch_cuda, n):
    T, D, F = 16, 8, 64
    W, FI = L.synth_ensemble(T, D, F, seed=950)
    x = L.synth_tuples(0, max(n, 1), F, seed=951)[:n]
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, leaves=True)
        for v in VARIANTS:
            e.set_kernel_variant(v)
            got = e.infer_host_leaves(x)
            assert got.shape == (n, T)
            if n:
                assert_words(got, leaf_cells(W, FI, x, D, L.MISSING_DEFAULT), "n=%d" % n)


def test_tile_edges_over_several_waves(torch_cuda):
    T, D, F = 24, 10, 256
    with make_engine(T, D, F) as e:
        W, FI = L.synth_ensemble(T, D, F, seed=960)
        FI = early(FI, D, 961)
        wl, fl = L.pack_streams(W, FI, D)
        e.load_ensemble(wl, fl, leaves=True)
        for v in (E.DTE_KERNEL_TILE, E.DTE_KERNEL_TILE_STAGED):
            e.set_kernel_variant(v)
            M = int(e.info()["tuples_per_cta"])
            for n in (3 * 132 * M - 1, 3 * 132 * M + 1, M - 1, M + 1):
                x = L.synth_tuples(0, n, F, seed=962, missing_ppm=20000)
                assert_words(device_leaves(torch_cuda, e, x, T), leaf_cells(W, FI, x, D, L.MISSING_DEFAULT), "n=%d" % n)


def test_trees_beyond_the_score_slots(torch_cuda):
    """Every resident tree is walked: K*S*8 = 8 slots, 21 trees."""
    run(torch_cuda, 21, 9, 32, 500, 970, K=1, S=1)


def test_classes_with_a_chunk_and_256_classes(torch_cuda):
    T, D, F, first, cnt = 40, 8, 32, 5, 29
    W, FI = L.synth_ensemble(T, D, F, seed=980)
    FI = early(FI, D, 981)
    x = L.synth_tuples(0, 900, F, seed=982, missing_ppm=20000)
    wl, fl = L.pack_streams(W, FI, D)
    want = leaf_cells(W[first:first + cnt], FI[first:first + cnt], x, D, L.MISSING_DEFAULT)
    with make_engine(T, D, F, K=1, S=1) as e:              # S*K*8 below the largest class: scores would refuse
        e.load_ensemble(wl, fl, first_tree=first, num_local_trees=cnt, num_classes=3, leaves=True)
        for v in VARIANTS:
            e.set_kernel_variant(v)
            assert_words(e.infer_host_leaves(x), want, "C=3 %s" % E.KERNEL_NAMES[v])
            assert_words(device_leaves(torch_cuda, e, x, cnt), want, "C=3 device %s" % E.KERNEL_NAMES[v])
    run(torch_cuda, 300, 6, 16, 300, 990, C=256, variants=[E.DTE_KERNEL_AUTO, E.DTE_KERNEL_GENERIC])


def test_scores_rebuilt_from_the_cells(torch_cuda):
    """leaf_values, then tree8 / slot / cluster order with the oracle's adder, equals the handle's own score words."""
    T, D, F, K, n = 37, 9, 64, 2, 600
    S = -(-T // (8 * K))
    W, FI = L.synth_ensemble(T, D, F, seed=1000)
    FI = early(FI, D, 1001)
    x = L.synth_tuples(0, n, F, seed=1002, missing_ppm=20000)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F, K, S) as e:
        e.load_ensemble(wl, fl, leaves=True)
        cells = device_leaves(torch_cuda, e, x, T)
        dx = torch_cuda.from_numpy(x.view(np.int32)).cuda()
        sc = torch_cuda.empty(n, dtype=torch_cuda.float32, device="cuda")
        e.infer_device(dx, n, sc)
        words = sc.cpu().numpy().view(np.uint32)
    v = np.zeros((n, S * K * 8), dtype=np.uint32)
    v[:, :T] = L.leaf_values(W, cells)
    add = O.fpadd_many
    tot = np.zeros(n, dtype=np.uint32)
    acc = [np.zeros(n, dtype=np.uint32) for _ in range(K)]
    for s in range(S):
        for j in range(K):
            l = v[:, (s * K + j) * 8: (s * K + j) * 8 + 8]
            r = add(add(add(l[:, 0], l[:, 1]), add(l[:, 2], l[:, 3])), add(add(l[:, 4], l[:, 5]), add(l[:, 6], l[:, 7])))
            acc[j] = add(r, acc[j])
    for j in range(K):
        tot = add(acc[j], tot)
    assert (tot == words).all()


def test_large_output_offset(torch_cuda):
    """A row past 4 GiB of output: the row offset is 64-bit."""
    T, D, F = 64, 6, 4
    free = torch_cuda.cuda.mem_get_info()[0]
    if free < (5 << 30):
        pytest.skip("needs 5 GiB of free device memory")
    W, FI = L.synth_ensemble(T, D, F, seed=1010)
    wl, fl = L.pack_streams(W, FI, D)
    n = (4 << 30) // (2 * T) + 1000
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, leaves=True)
        dx = torch_cuda.empty((n, F), dtype=torch_cuda.int32, device="cuda")
        e.synth_tuples_device(dx, 0, n, F, 5, 20000, L.MISSING_DEFAULT)
        out = torch_cuda.empty(n * T, dtype=torch_cuda.int16, device="cuda")
        e.infer_device_leaves(dx, n, out)
        tail = out[(n - 500) * T:].cpu().numpy().view(np.uint16).reshape(500, T)
        x = L.synth_tuples(n - 500, 500, F, seed=5, missing_ppm=20000)
        assert_words(tail, leaf_cells(W, FI, x, D, L.MISSING_DEFAULT), "rows past 4 GiB")
        del out, dx


def test_ordered_with_torch_work_on_a_stream(torch_cuda):
    T, D, F, n = 16, 8, 32, 5000
    W, FI = L.synth_ensemble(T, D, F, seed=1020)
    x = L.synth_tuples(0, n, F, seed=1021)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, leaves=True)
        s = torch_cuda.cuda.Stream()
        host = torch_cuda.from_numpy(x.view(np.int32)).pin_memory()
        with torch_cuda.cuda.stream(s):
            dx = host.to("cuda", non_blocking=True)            # the tuples arrive on s, the walk must wait for them
            out = torch_cuda.zeros(n * T, dtype=torch_cuda.int16, device="cuda")
            e.infer_device_leaves(dx, n, out, stream=s.cuda_stream)
            got = out.view(n, T).to("cpu", non_blocking=True)
        s.synchronize()
        assert_words(got.numpy().view(np.uint16), leaf_cells(W, FI, x, D, L.MISSING_DEFAULT), "stream")


def test_refusals_and_binned_load(torch_cuda):
    T, D, F, n = 16, 8, 32, 64
    W, FI = L.synth_ensemble(T, D, F, seed=1030, cuts=16)
    x = L.synth_tuples(0, n, F, seed=1031)
    wl, fl = L.pack_streams(W, FI, D)
    dx = torch_cuda.from_numpy(x.view(np.int32)).cuda()
    out = torch_cuda.empty(n * T + 16, dtype=torch_cuda.int16, device="cuda")
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl)                            # no leaf layout
        for call in (lambda: e.infer_host_leaves(x), lambda: e.infer_device_leaves(dx, n, out), e.kernel_name_leaves):
            refused(call, E.DTE_ERR_STATE)
        base = e.info()["ensemble_bytes"]
        e.load_ensemble(wl, fl, leaves=True)
        assert e.info()["ensemble_bytes"] > base
        for bad_x, bad_o in ((dx.view(-1)[1:], out), (dx, out[1:]), (dx, out[4:])):
            refused(lambda: e.infer_device_leaves(bad_x, n - 1, bad_o), E.DTE_ERR_ARG)
        e.load_ensemble(wl, fl, binned=True, leaves=True)  # a binned load with the option on answers the fp32 leaf calls
        assert_words(e.infer_host_leaves(x), leaf_cells(W, FI, x, D, L.MISSING_DEFAULT), "binned load")
        e.load_ensemble(wl, fl)                            # a placement without the option drops the layout
        refused(lambda: e.infer_host_leaves(x), E.DTE_ERR_STATE)
        assert e.info()["ensemble_bytes"] == base


def test_line_stream_placement(torch_cuda):
    """A tree line stream after `start` places the leaf layout while the option is on."""
    T, D, F, n = 16, 7, 16, 300
    W, FI = L.synth_ensemble(T, D, F, seed=1040)
    FI = early(FI, D, 1041)
    x = L.synth_tuples(0, n, F, seed=1042)
    wl, fl = L.pack_streams(W, FI, D)
    with ddt.Engine(0) as e:
        e.configure(T, D, 4 * F, clusters=2, n_tuples=n)
        e.set_option(E.DTE_OPT_LEAF_LAYOUT, 1)
        e.start()
        e.stream_write(wl)
        e.stream_write(fl)
        e.stream_write(x)
        e.stream_flush()
        assert_words(e.infer_host_leaves(x), leaf_cells(W, FI, x, D, L.MISSING_DEFAULT), "line stream")


@pytest.mark.parametrize("mode", ["data", "ensemble"])
def test_multi_device_handles(torch_cuda, mode):
    """[0, 0, 0]: Dealt rows in global tuple order; Chunked columns of every ring position."""
    T, D, F, K, n = 44, 8, 32, 2, 2000
    W, FI = L.synth_ensemble(T, D, F, seed=1050)
    FI = early(FI, D, 1051)
    x = L.synth_tuples(0, n, F, seed=1052, missing_ppm=20000)
    wl, fl = L.pack_streams(W, FI, D)
    want = leaf_cells(W, FI, x, D, L.MISSING_DEFAULT)
    with ddt.Engine([0, 0, 0]) as e:
        write_regs(e, multi_node_regs(T, D, F, K, n, 3, mode))
        e.set_option(E.DTE_OPT_CHUNK_TUPLES, 256)
        e.load_ensemble(wl, fl, leaves=True)
        for v in (E.DTE_KERNEL_AUTO, E.DTE_KERNEL_GENERIC):
            e.set_kernel_variant(v)
            assert_words(e.infer_host_leaves(x), want, "%s %s" % (mode, E.KERNEL_NAMES[v]))


def test_headline_leaf_plan_multi_tile(torch_cuda):
    """cfg3's geometry (D = 12, F = 256) on the AUTO plan, the phased staged leaf walk, with three tiles per CTA."""
    T, D, F = 64, 12, 256
    W, FI = L.synth_ensemble(T, D, F, seed=1060)
    FI = early(FI, D, 1061)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, leaves=True)
        name = e.kernel_name_leaves()
        print("shipped-plan leaf kernel:", name)
        assert name.startswith("dt_walk_tile_leaf<4, 2, 1, 0, 384>") and "phased=1" in name, name
        n = 3 * 132 * int(e.info()["tuples_per_cta"]) - 5
        x = L.synth_tuples(0, n, F, seed=1062, missing_ppm=20000)
        assert_words(device_leaves(torch_cuda, e, x, T), leaf_cells(W, FI, x, D, L.MISSING_DEFAULT), name)


def test_many_trees_few_features(torch_cuda):
    """2048 trees on 4 features: a tuple's cells (4 KiB) are 256 times its bytes, so the leaf run lands fewer tuples per
    slot (at most twice the tuple budget in cells) and the rows of several slots must still come back in order."""
    T, D, F, n = 2048, 4, 4, 70000
    W, FI = L.synth_ensemble(T, D, F, seed=1070)
    x = L.synth_tuples(0, n, F, seed=1071, missing_ppm=20000)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F) as e:
        e.load_ensemble(wl, fl, leaves=True)
        assert_words(e.infer_host_leaves(x), leaf_cells(W, FI, x, D, L.MISSING_DEFAULT), "T=2048, F=4")

