"""Sparse tuples on the H100 (DESIGN.md §11): CSR rows whose absent features take the `absent` word.

Bar everywhere: every score word and label equals the dense walk of the same handle on the rows tests/sparse_ref.py
densifies, and a sample also equals the oracle on those rows."""
import numpy as np
import pytest

import ddt_b200 as ddt
from ddt_b200 import engine as E
from edge_operands import edge_ensemble, edge_tuples
from helpers import (assert_words, geometry_regs, make_engine, multi_node_regs, oracle_words, refused, torch_cuda,
                     write_regs, L)  # noqa: F401 (torch_cuda: a fixture)
from sparse_ref import densify, density_mask, sparse_rows

pytestmark = pytest.mark.gpu

VARIANTS = [E.DTE_KERNEL_GENERIC, E.DTE_KERNEL_TILE, E.DTE_KERNEL_TILE_STAGED, E.DTE_KERNEL_AUTO]


def assert_same(got, want, what):
    """(scores, labels) against (scores, labels), word for word."""
    assert_words(got[0], want[0], what + ": scores")
    assert_words(got[1], want[1], what + ": labels")


def to_device(torch, indptr, indices, values):
    out = (torch.from_numpy(indptr).cuda(), torch.from_numpy(indices.view(np.int32)).cuda(),
           torch.from_numpy(values.view(np.int32)).cuda())
    torch.cuda.synchronize()
    return out


def device_scores(torch, e, rows, n, C, absent=None):
    """infer_device_sparse on the engine's own stream (a synchronous call) -> (scores, labels)."""
    d_ptr, d_idx, d_val = to_device(torch, *rows)
    ds = torch.empty((n, C) if C > 1 else (n,), dtype=torch.float32, device="cuda")
    dl = torch.empty(n, dtype=torch.uint8, device="cuda")
    e.infer_device_sparse(d_ptr, d_idx, d_val, n, ds, dl, absent=absent)
    return ds.cpu().numpy(), dl.cpu().numpy()


def pinned_copy(e, a):
    """a copy of `a` in host_alloc memory (release with e.host_free)."""
    p = e.host_alloc((max(1, a.size),), a.dtype)[: a.size]
    p[:] = a
    return p


def run_case(torch, T, D, F, K, S, C, n, density, seed, variants=VARIANTS):
    """Sparse rows made from synthetic tuples at `density`, absent = the missing pattern: host and device sparse calls
    against the dense walk of the densified rows on every variant, and the first 512 rows against the oracle."""
    W, FI = L.synth_ensemble(T, D, F, seed=seed)
    x = L.synth_tuples(0, n, F, seed=seed + 1, missing_ppm=20000)
    rows = sparse_rows(x, density_mask(n, F, density, seed + 2), seed + 3, base=3)
    dense = densify(*rows, F, L.MISSING_DEFAULT)
    want = oracle_words(W, FI, dense[:512], D, K, S, C, L.MISSING_DEFAULT)
    with make_engine(T, D, F, K, S) as e:
        e.load_ensemble(*L.pack_streams(W, FI, D), num_classes=C)
        for v in variants:
            e.set_kernel_variant(v)
            name = E.KERNEL_NAMES[v]
            ref = e.infer_host(dense)
            assert (ref[0].view(np.uint32)[:512] == want).all(), "dense walk against the oracle, " + name
            assert_same(e.infer_host_sparse(rows), ref, "host sparse, %s, density %g" % (name, density))
            assert_same(device_scores(torch, e, rows, n, C), ref, "device sparse, %s, density %g" % (name, density))


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("density", [0.0, 0.01, 0.1, 1.0])
def test_densities_and_classes(torch_cuda, density, C):
    run_case(torch_cuda, 48, 8, 132, 2, 3 if C == 1 else 1, C, 2001, density, 100 + int(density * 100) + C)


@pytest.mark.parametrize("F", [20, 516])
def test_feature_counts(torch_cuda, F):
    run_case(torch_cuda, 24, 7, F, 2, 2, 1, 1501, 0.1, 200 + F)


def test_edge_operands_absent_where_missing(torch_cuda):
    """Edge tuples whose every missing-pattern cell becomes an absence give the dense edge rows' words; then, after a
    reg-205 write that changes the pattern: DTE_SPARSE_ABSENT_MISSING follows the new pattern, absent = 0 gives zeros,
    and explicit entries equal to the new pattern are missing."""
    torch = torch_cuda
    T, D, F, K, S, n, m = 40, 7, 36, 1, 5, 3001, 0x80000000
    W, FI, pools = edge_ensemble(T, D, F, 300, leaves="wide", missing=m)
    x = edge_tuples(n, F, pools, 301, m)
    rows = sparse_rows(x, x != m, 302)
    with make_engine(T, D, F, K, S, m) as e:
        e.load_ensemble(*L.pack_streams(W, FI, D))
        want = oracle_words(W, FI, x, D, K, S, 1, m)
        ref = e.infer_host(x)
        assert (ref[0].view(np.uint32) == want).all()
        assert_same(e.infer_host_sparse(rows), ref, "edge rows, host")
        assert_same(device_scores(torch, e, rows, n, 1), ref, "edge rows, device")
        m2 = 0x7FC00000
        e.softreg_write(205, (geometry_regs(T, D, F, K, S, m)[205] & ~0xFFFFFFFF) | m2)
        xm = x.copy()
        xm[:, ::5] = m2                                       # explicit entries equal to the new pattern
        rows2 = sparse_rows(xm, x != m, 303)
        for absent, word in ((None, m2), (0, 0), (m, m)):
            dense = densify(*rows2, F, word)
            ref = e.infer_host(dense)
            assert (ref[0].view(np.uint32)[:300] == oracle_words(W, FI, dense[:300], D, K, S, 1, m2)).all()
            assert_same(e.infer_host_sparse(rows2, absent=absent), ref, "host, absent %r" % absent)
            assert_same(device_scores(torch, e, rows2, n, 1, absent=absent), ref, "device, absent %r" % absent)


def test_sparse_to_dense_device_bytes(torch_cuda):
    """Byte for byte the reference rows, from a row slice of larger arrays (indptr[0] != 0), on a side stream."""
    torch = torch_cuda
    T, D, F, n = 8, 4, 132, 3001
    x = L.synth_tuples(0, n, F, seed=400)
    rows = sparse_rows(x, density_mask(n, F, 0.3, 401), 402, base=17)
    with make_engine(T, D, F, 1, 1) as e:
        d_ptr, d_idx, d_val = to_device(torch, *rows)
        for absent, word in ((None, L.MISSING_DEFAULT), (0, 0), (0x12345678, 0x12345678)):
            out = torch.full((n, F), -1, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            s = torch.cuda.Stream()
            e.sparse_to_dense_device(d_ptr, d_idx, d_val, n, out, absent=absent, stream=s.cuda_stream)
            s.synchronize()
            assert (out.cpu().numpy().view(np.uint32) == densify(*rows, F, word)).all(), absent
        # a row slice: rows 100.. of the same arrays, indices still absolute
        d_ptr, d_idx, d_val = to_device(torch, *rows)
        out = torch.empty((n - 100, F), dtype=torch.int32, device="cuda")
        e.sparse_to_dense_device(d_ptr[100:], d_idx, d_val, n - 100, out, absent=0)
        assert (out.cpu().numpy().view(np.uint32) == densify(rows[0][100:], rows[1], rows[2], F, 0)).all()


def test_sparse_to_dense_device_past_4_gib(torch_cuda):
    """F = 256 and 4.2 M mostly empty rows: 4.3 GB of output, rows with entries on both sides of 4 GiB."""
    torch = torch_cuda
    F, n = 256, 4_200_000
    assert n * F * 4 > 2 ** 32
    full = [0, 1, 77, 4_194_303, 4_194_304, 4_194_305, n - 2, n - 1]      # row 4194304 starts at byte 2^32
    x = L.synth_tuples(0, len(full), F, seed=500)
    sub = sparse_rows(x, density_mask(len(full), F, 0.5, 501), 502)
    counts = np.zeros(n, dtype=np.int64)
    counts[full] = np.diff(sub[0])
    indptr = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    with make_engine(8, 4, F, 1, 1) as e:
        out = torch.empty((n, F), dtype=torch.int32, device="cuda")
        d_ptr, d_idx, d_val = to_device(torch, indptr, sub[1], sub[2])
        e.sparse_to_dense_device(d_ptr, d_idx, d_val, n, out, absent=0x3F800000)
        torch.cuda.synchronize()
        got = out[torch.tensor(full, device="cuda")].cpu().numpy().view(np.uint32)
        assert (got == densify(*sub, F, 0x3F800000)).all()
        out[torch.tensor(full, device="cuda")] = 0x3F800000
        assert bool((out == 0x3F800000).all())
        del out


@pytest.mark.parametrize("n", [0, 1, 7, 5003])
def test_host_counts_pinned_pageable_scipy(torch_cuda, n):
    """n = 0, 1, not a multiple of 4, and several landing slots (DTE_OPT_CHUNK_TUPLES = 1000); pinned (host_alloc) and
    pageable sources, and a scipy csr_matrix passed as it is."""
    T, D, F, K, S = 32, 6, 132, 2, 2
    W, FI = L.synth_ensemble(T, D, F, seed=600)
    x = L.synth_tuples(0, n, F, seed=601, missing_ppm=20000)
    rows = sparse_rows(x, density_mask(n, F, 0.1, 602), 603)
    with make_engine(T, D, F, K, S) as e:
        e.set_option(E.DTE_OPT_CHUNK_TUPLES, 1000)
        e.load_ensemble(*L.pack_streams(W, FI, D))
        ref = e.infer_host(densify(*rows, F, L.MISSING_DEFAULT))
        assert_same(e.infer_host_sparse(rows), ref, "pageable")
        pinned = [pinned_copy(e, a) for a in rows]
        assert_same(e.infer_host_sparse(tuple(pinned)), ref, "pinned")
        for p in pinned:
            e.host_free(p)
        sp = pytest.importorskip("scipy.sparse")
        dense = np.where(density_mask(n, F, 0.1, 604), x.view(np.float32), np.float32(0))
        m = sp.csr_matrix(dense)
        ref0 = e.infer_host(dense.astype(np.float32))
        assert_same(e.infer_host_sparse(m, absent=0), ref0, "scipy csr_matrix, absent 0")


def test_host_pageable_staging_and_many_slots(torch_cuda):
    """Arrays of over 256 KiB go through the pageable staging ring; n spans eleven landing slots."""
    T, D, F, K, S, n = 32, 8, 132, 2, 2, 40_000
    W, FI = L.synth_ensemble(T, D, F, seed=650)
    x = L.synth_tuples(0, n, F, seed=651, missing_ppm=20000)
    rows = sparse_rows(x, density_mask(n, F, 0.2, 652), 653, extras=False)
    assert rows[1].nbytes > 256 << 10
    with make_engine(T, D, F, K, S) as e:
        e.set_option(E.DTE_OPT_CHUNK_TUPLES, 3700)
        e.load_ensemble(*L.pack_streams(W, FI, D))
        ref = e.infer_host(np.where(density_mask(n, F, 0.2, 652), x, np.uint32(L.MISSING_DEFAULT)))
        info = e.info()
        assert_same(e.infer_host_sparse(rows), ref, "pageable, many slots")
        after = e.info()
        assert after["tuples_in"] - info["tuples_in"] == n and after["tuples_out"] - info["tuples_out"] == n
        assert after["last_walk_ms"] > 0


@pytest.mark.parametrize("mode", ["data", "ensemble"])
def test_multi_device_handles(torch_cuda, mode):
    """Dealt and Chunked handles with three ring positions on one GPU: the sparse words equal the handle's dense words,
    and Dealt's also the single handle's."""
    T, D, F, K, n, G = 44, 8, 36, 2, 7001, 3
    W, FI = L.synth_ensemble(T, D, F, seed=700)
    x = L.synth_tuples(0, n, F, seed=701, missing_ppm=20000)
    rows = sparse_rows(x, density_mask(n, F, 0.3, 702), 703, base=9)
    dense = densify(*rows, F, L.MISSING_DEFAULT)
    wl, fl = L.pack_streams(W, FI, D)
    regs = multi_node_regs(T, D, F, K, n, G, mode, batch_tuples=64)
    with ddt.Engine([0] * G) as e:
        e.set_option(E.DTE_OPT_CHUNK_TUPLES, 900)
        write_regs(e, regs)
        e.load_ensemble(wl, fl)
        ref = e.infer_host(dense)
        for _ in range(2):
            assert_same(e.infer_host_sparse(rows), ref, mode)
        pinned = [pinned_copy(e, a) for a in rows]
        assert_same(e.infer_host_sparse(tuple(pinned)), ref, mode + ", pinned")
        for p in pinned:
            e.host_free(p)
        assert_same(e.infer_host(dense), ref, mode + ", dense after sparse")
        for call in (lambda: e.infer_device_sparse(0, 0, 0, 0, 0), lambda: e.sparse_to_dense_device(0, 0, 0, 0, 0)):
            refused(call, E.DTE_ERR_UNSUPPORTED)
    if mode == "data":
        S = (regs[205] >> 36) & 0xFF
        with make_engine(T, D, F, K, S) as e:
            e.load_ensemble(wl, fl)
            assert_same(e.infer_host(dense), ref, "single handle")


def test_device_side_stream_and_chunks(torch_cuda):
    """infer_device_sparse on a torch side stream over several chunks (both scratch buffers in turn, twice), a C = 3
    ensemble; correct once the stream has synchronised, and counted like infer_device."""
    torch = torch_cuda
    T, D, F, K, S, C, n = 48, 8, 64, 2, 1, 3, 5003
    W, FI = L.synth_ensemble(T, D, F, seed=800)
    x = L.synth_tuples(0, n, F, seed=801, missing_ppm=20000)
    rows = sparse_rows(x, density_mask(n, F, 0.1, 802), 803)
    with make_engine(T, D, F, K, S) as e:
        e.set_option(E.DTE_OPT_CHUNK_TUPLES, 1200)
        e.load_ensemble(*L.pack_streams(W, FI, D), num_classes=C)
        ref = e.infer_host(densify(*rows, F, L.MISSING_DEFAULT))
        d_ptr, d_idx, d_val = to_device(torch, *rows)
        torch.cuda.synchronize()
        info = e.info()
        for _ in range(2):
            s = torch.cuda.Stream()
            ds = torch.empty((n, C), dtype=torch.float32, device="cuda")
            dl = torch.empty(n, dtype=torch.uint8, device="cuda")
            e.infer_device_sparse(d_ptr, d_idx, d_val, n, ds, dl, stream=s.cuda_stream)
            s.synchronize()
            assert_same((ds.cpu().numpy(), dl.cpu().numpy()), ref, "side stream")
        after = e.info()
        assert after["tuples_in"] - info["tuples_in"] == 2 * n and after["tuples_out"] - info["tuples_out"] == 2 * n
        assert after["last_walk_ms"] > 0


def test_refusals_before_any_launch(torch_cuda):
    torch = torch_cuda
    T, D, F, K, S, n = 16, 5, 16, 1, 2, 64
    W, FI = L.synth_ensemble(T, D, F, seed=900)
    x = L.synth_tuples(0, n, F, seed=901)
    wl, fl = L.pack_streams(W, FI, D)
    rows = sparse_rows(x, density_mask(n, F, 0.5, 902), 903)
    with make_engine(T, D, F, K, S) as e:
        refused(lambda: e.infer_host_sparse(rows), E.DTE_ERR_STATE)        # no ensemble
        e.load_ensemble(wl, fl)
        info = e.info()
        p, i, v = to_device(torch, *rows)
        big = torch.zeros(n * F + 16, dtype=torch.float32, device="cuda")
        sc = torch.zeros(n + 4, dtype=torch.float32, device="cuda")
        P, I, V, B, SC = p.data_ptr(), i.data_ptr(), v.data_ptr(), big.data_ptr(), sc.data_ptr()
        for args in ((P + 4, I, V), (P, I + 2, V), (P, I, V + 2)):
            for call in (lambda a: e.infer_device_sparse(*a, n, SC), lambda a: e.sparse_to_dense_device(*a, n, B)):
                refused(lambda: call(args), E.DTE_ERR_ARG, "aligned")
        for call in (lambda: e.infer_device_sparse(P, I, V, n, SC + 2), lambda: e.sparse_to_dense_device(P, I, V, n, B + 4),
                     lambda: e.infer_device_sparse(P, I, V, n, SC, absent=2 ** 32)):
            refused(call, E.DTE_ERR_ARG)
        hp, hi, hv = rows
        raw = np.zeros(hp.size + 1, dtype=np.int64)
        mis = raw.view(np.uint8)[4:4 + 8 * hp.size].view(np.int64)       # 4 bytes off an 8-byte boundary
        mis[:] = hp
        fn = e._lib.dte_infer_host_sparse
        out = np.empty(n, np.float32)
        assert fn(e._h, E._ptr(mis), E._ptr(hi), E._ptr(hv), n, E.DTE_SPARSE_ABSENT_MISSING, E._ptr(out), None) == E.DTE_ERR_ARG
        bad = hp.copy()
        bad[40] = bad[39] - 1
        refused(lambda: e.infer_host_sparse((bad, hi, hv)), E.DTE_ERR_ARG, "row 39")
        refused(lambda: e.infer_host_sparse(rows, absent=2 ** 40), E.DTE_ERR_ARG)
        after = e.info()
        assert after["kernel_launches"] == info["kernel_launches"] and after["tuples_in"] == info["tuples_in"]
        # a partial tuple pending in the line stream
        e.configure(T, D, 4 * F, clusters=K, n_tuples=n)
        e.start()
        e.stream_write(wl)
        e.stream_write(fl)
        e.stream_write(x.reshape(-1, 4)[:5])                  # one tuple and a quarter
        refused(lambda: e.infer_host_sparse(rows), E.DTE_ERR_STATE)


def test_dense_binned_and_leaf_calls_after_sparse(torch_cuda):
    """A sparse host call leaves no landing slot partly filled: the dense, binned and leaf host calls right after it give
    the words and cells they gave before it."""
    T, D, F, K, S, n = 40, 8, 64, 2, 3, 4001
    W, FI = L.synth_ensemble(T, D, F, seed=1000, cuts=64)
    x = L.synth_tuples(0, n, F, seed=1001, missing_ppm=20000)
    rows = sparse_rows(x, density_mask(n, F, 0.1, 1002), 1003)
    with make_engine(T, D, F, K, S) as e:
        e.set_option(E.DTE_OPT_CHUNK_TUPLES, 1500)
        e.load_ensemble(*L.pack_streams(W, FI, D), binned=True, leaves=True)
        b = L.bin_tuples(x, *e.bin_edges())
        dense, binned, leaves = e.infer_host(x), e.infer_host_binned(b), e.infer_host_leaves(x)
        assert (dense[0].view(np.uint32) == oracle_words(W, FI, x, D, K, S, 1, L.MISSING_DEFAULT)).all()
        for _ in range(2):
            assert_same(e.infer_host_sparse(rows), e.infer_host(densify(*rows, F, L.MISSING_DEFAULT)), "sparse")
            e.infer_host_sparse((rows[0][:1001], rows[1], rows[2]))        # ends mid-slot
            assert_same(e.infer_host(x), dense, "dense after sparse")
            e.infer_host_sparse((rows[0][:1001], rows[1], rows[2]))
            assert_same(e.infer_host_binned(b), binned, "binned after sparse")
            e.infer_host_sparse((rows[0][:1001], rows[1], rows[2]))
            assert (e.infer_host_leaves(x) == leaves).all(), "leaves after sparse"
