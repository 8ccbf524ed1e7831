"""Multi-class ensembles (dte_load_ensemble_classes): one walk returns [n][C] scores and argmax labels.

Bar: score[i][c] is bit for bit the oracle's score of the class-c trees alone (stream tree t belongs to class t % C) —
which is also what a single-class handle loaded with W[c::C] returns — and label[i] is the first class of maximal
score (numpy argmax).  Every kernel variant and launch plan, the device-pointer paths, and both multi-device
partitions are covered; the oracle needs no new arithmetic (oracle_class_scores below composes per-class O.scores)."""
import ctypes as C
import os

import numpy as np
import pytest

import ddt_b200 as ddt
from ddt_b200 import engine as E
from helpers import labels_of, make_engine, multi_node_regs, oracle_scores, refused, torch_cuda, write_regs, L  # noqa: F401
from oracle import oracle as O

pytestmark = pytest.mark.gpu

VARIANTS = [E.DTE_KERNEL_GENERIC, E.DTE_KERNEL_TILE, E.DTE_KERNEL_TILE_STAGED, E.DTE_KERNEL_AUTO]


def oracle_class_scores(W, FI, x, D, K, S, missing, C, tree_range=None):
    """Multi-class oracle: uint32 words [n, C], column c = O.scores of the class-c trees alone (stream tree t belongs to
    class t % C), in stream order.  tree_range = (first, count) restricts to the trees of one chunk (a ring position's
    per-class partials); a class with no tree there scores +0."""
    first, count = tree_range if tree_range is not None else (0, W.shape[0])
    out = np.zeros((x.shape[0], C), dtype=np.uint32)
    for c in range(C):
        idx = [t for t in range(first, first + count) if t % C == c]
        if idx:
            out[:, c] = oracle_scores(W[idx], FI[idx], x, D, K, S, missing)
    return out


def slots_for(T, nc, K):
    """Smallest S whose S*K*8 slots hold the largest class."""
    return -(-(-(-T // nc)) // (8 * K))


def check_mc(W, FI, x, D, K, S, nc, variants=VARIANTS, singles=True):
    T, F, n = W.shape[0], x.shape[1], x.shape[0]
    wl, fl = L.pack_streams(W, FI, D)
    want = oracle_class_scores(W, FI, x, D, K, S, L.MISSING_DEFAULT, nc)
    with make_engine(T, D, F, K, S) as e:
        e.load_ensemble(wl, fl, num_classes=nc)
        assert e.info()["num_classes"] == nc and e.kernel_name().endswith(" classes=%d" % nc)
        for v in variants:
            e.set_kernel_variant(v)
            sc, lb = e.infer_host(x)
            assert sc.shape == (n, nc)
            got = sc.view(np.uint32)
            bad = np.argwhere(got != want)
            assert bad.size == 0, "variant %s (%s): %d words differ, first at %s" % (E.KERNEL_NAMES[v], e.kernel_name(), len(bad), bad[0])
            assert (lb == labels_of(want, nc)).all()
    if singles:
        # the same words from C single-class handles, each loaded with every C-th tree
        for c in range(nc):
            wc, fc = L.pack_streams(W[c::nc], FI[c::nc], D)
            with make_engine(W[c::nc].shape[0], D, F, K, S) as e1:
                e1.load_ensemble(wc, fc)
                s1, _ = e1.infer_host(x)
                assert (s1.view(np.uint32) == want[:, c]).all(), c
    return want


@pytest.mark.parametrize("D,T,F,K,nc,n", [
    (1, 23, 8, 1, 2, 300),          # D = 1 extension
    (4, 50, 32, 2, 3, 1000),
    (7, 95, 64, 4, 10, 2000),
    (12, 31, 256, 8, 3, 900),       # headline depth and width
    (6, 44, 600, 2, 3, 700),        # wide feature indexes (64-byte records)
    (9, 203, 128, 8, 10, 1500),     # several groups per class
])
def test_random_multiclass_ensembles_bit_exact(D, T, F, K, nc, n):
    assert T % nc != 0
    W, FI = L.synth_ensemble(T, D, F, seed=3000 + D + nc)
    x = L.synth_tuples(0, n, F, seed=3100 + D, missing_ppm=20000)
    check_mc(W, FI, x, D, K, slots_for(T, nc, K), nc)


@pytest.mark.parametrize("tune", ["pair=1,ilp=8,stages=1", "pair=1,ilp=4,stages=2", "pair=2,stages=1", "pair=2,stages=2",
                                  "pair=4,stages=1", "pair=1,ilp=8,stages=2,warps=3", "pair=2,stages=1,warps=4",
                                  "pair=2,ilp=2,stages=2", "pair=2,stages=1,phased=1", "pair=1,ilp=8,stages=1,phased=1",
                                  "pair=4,stages=2,phased=1"])
def test_every_launch_plan_multiclass(tune, monkeypatch):
    """Every DTE_TUNE plan of the single-class plan test, with three classes (uneven: 24 / 23 / 23 trees)."""
    monkeypatch.setenv("DTE_TUNE", tune)
    W, FI = L.synth_ensemble(70, 9, 64, seed=3201)
    x = L.synth_tuples(0, 1500, 64, seed=3202, missing_ppm=20000)
    check_mc(W, FI, x, 9, 4, 1, 3, variants=[E.DTE_KERNEL_TILE_STAGED, E.DTE_KERNEL_TILE], singles=False)
    W, FI = L.synth_ensemble(49, 12, 256, seed=3203)        # the headline geometry, 17 / 16 / 16 trees
    x = L.synth_tuples(0, 700, 256, seed=3204)
    check_mc(W, FI, x, 12, 8, 1, 3, variants=[E.DTE_KERNEL_TILE_STAGED], singles=False)


def test_multiclass_headline_geometry_multi_tile(capsys):
    """The shipped plan for D = 12, F = 256 with C = 3, on enough tuples that every persistent CTA walks several tiles.
    tools/gpu_sanitize.sh runs this case under compute-sanitizer (memcheck, synccheck)."""
    T, D, F, K, nc = 50, 12, 256, 8, 3
    n = 160 * 132 * 2 + 77
    if os.environ.get("DTE_TEST_SANITIZER"):          # instrumented runs: fewer trees, CTAs 0..2 still walk two tiles
        T, n = 22, 160 * 132 + 333
    W, FI = L.synth_ensemble(T, D, F, seed=3301)
    x = L.synth_tuples(0, n, F, seed=3302, missing_ppm=15000)
    S = slots_for(T, nc, K)
    wl, fl = L.pack_streams(W, FI, D)
    want = oracle_class_scores(W, FI, x, D, K, S, L.MISSING_DEFAULT, nc)
    with make_engine(T, D, F, K, S) as e:
        e.load_ensemble(wl, fl, num_classes=nc)
        name = e.kernel_name()
        with capsys.disabled():
            print("\n[multiclass-plan] DTE_TUNE=%r -> %s" % (os.environ.get("DTE_TUNE", ""), name))
        sc, lb = e.infer_host(x)
        assert e.info()["tuples_per_cta"] * e.info()["sm_count"] < n
    assert (sc.view(np.uint32) == want).all() and (lb == labels_of(want, nc)).all()


def test_device_pointer_path_and_accumulate(torch_cuda):
    """dte_infer_device on a torch stream writes [n][C] and argmax labels; accumulating into a zeroed buffer gives the
    same words (+0 + s = s)."""
    torch = torch_cuda
    T, D, F, K, nc, n = 58, 8, 128, 4, 3, 5000
    W, FI = L.synth_ensemble(T, D, F, seed=3401)
    x = L.synth_tuples(0, n, F, seed=3402, missing_ppm=10000)
    S = slots_for(T, nc, K)
    wl, fl = L.pack_streams(W, FI, D)
    want = oracle_class_scores(W, FI, x, D, K, S, L.MISSING_DEFAULT, nc)
    st = torch.cuda.Stream()
    with make_engine(T, D, F, K, S) as e, torch.cuda.stream(st):
        e.load_ensemble(wl, fl, num_classes=nc)
        dx = torch.from_numpy(x.view(np.int32)).cuda()
        ds = torch.full((n, nc), float("nan"), dtype=torch.float32, device="cuda")
        dl = torch.full((n,), 255, dtype=torch.uint8, device="cuda")
        acc = torch.zeros((n, nc), dtype=torch.float32, device="cuda")
        e.infer_device(dx, n, ds, dl, stream=st.cuda_stream)
        e.infer_device_accumulate(dx, n, acc, stream=st.cuda_stream)
        st.synchronize()
        got = ds.cpu().numpy().view(np.uint32)
        assert (got == want).all()
        assert (dl.cpu().numpy() == labels_of(want, nc)).all()
        assert (acc.cpu().numpy().view(np.uint32) == want).all()
        # the device-side argmax over the same matrix
        dl2 = torch.zeros(n, dtype=torch.uint8, device="cuda")
        e.class_labels_device(ds, n, nc, dl2, stream=st.cuda_stream)
        st.synchronize()
        assert (dl2.cpu().numpy() == labels_of(want, nc)).all()


def test_ties_go_to_the_lower_class():
    """Classes with identical trees tie on every tuple: the label is the lower class.  C = 3 with class 0 = class 1
    negated (every leaf's sign flipped: round-to-nearest-even is symmetric, so its score is exactly the negation) and
    class 2 = class 1: label 1 where the shared score is > 0, else 0."""
    D, F, K, n, per = 6, 32, 2, 2000, 9
    B, FIb = L.synth_ensemble(per, D, F, seed=3501)
    x = L.synth_tuples(0, n, F, seed=3502, missing_ppm=10000)
    # C = 2: trees 2k and 2k + 1 identical
    W2, FI2 = np.repeat(B, 2, axis=0), np.repeat(FIb, 2, axis=0)
    want = check_mc(W2, FI2, x, D, K, slots_for(W2.shape[0], 2, K), 2, variants=[E.DTE_KERNEL_AUTO, E.DTE_KERNEL_GENERIC], singles=False)
    assert (want[:, 0] == want[:, 1]).all()
    # C = 3: class 0 negated, classes 1 and 2 identical
    neg = B.copy()
    neg[:, (1 << D) - 1:] ^= np.uint32(0x80000000)
    W3 = np.stack([neg, B, B], axis=1).reshape(3 * per, -1)
    FI3 = np.repeat(FIb, 3, axis=0)
    want = check_mc(W3, FI3, x, D, K, slots_for(W3.shape[0], 3, K), 3, variants=[E.DTE_KERNEL_AUTO, E.DTE_KERNEL_GENERIC], singles=False)
    s1 = want[:, 1].view(np.float32)
    assert (want[:, 1] == want[:, 2]).all() and (s1 > 0).any() and (s1 < 0).any()
    assert (labels_of(want, 3) == np.where(s1 > 0, 1, 0)).all()


def test_one_class_through_the_new_call_is_the_old_call():
    """dte_load_ensemble_classes(..., 1) = dte_load_ensemble: same words, labels and kernel name."""
    T, D, F, K, n = 45, 10, 256, 8, 1200
    W, FI = L.synth_ensemble(T, D, F, seed=3601)
    x = L.synth_tuples(0, n, F, seed=3602)
    wl, fl = L.pack_streams(W, FI, D)
    S = -(-T // (8 * K))
    out = []
    for new_call in (False, True):
        with make_engine(T, D, F, K, S) as e:
            if new_call:
                rc = e._lib.dte_load_ensemble_classes(e._h, wl.ctypes.data, wl.nbytes // 16, fl.ctypes.data, fl.nbytes // 16, 0, 0, 1)
                assert rc == 0
            else:
                e.load_ensemble(wl, fl)
            assert e.info()["num_classes"] == 1
            res = [e.kernel_name()]
            for v in VARIANTS:
                e.set_kernel_variant(v)
                sc, lb = e.infer_host(x)
                assert sc.shape == (n,)
                res += [sc.view(np.uint32).copy(), lb.copy()]
            out.append(res)
    assert out[0][0] == out[1][0] and "classes" not in out[0][0]
    for a, b in zip(out[0][1:], out[1][1:]):
        assert (a == b).all()
    assert (out[0][1] == oracle_scores(W, FI, x, D, K, S, L.MISSING_DEFAULT)).all()


def _mc_ring_reference(W, FI, x, D, K, S, nc, G):
    """Per ring position, per class oracle partials (contiguous tree chunks in ring order), combined word by word."""
    T = W.shape[0]
    parts = [oracle_class_scores(W, FI, x, D, K, S, L.MISSING_DEFAULT, nc, tree_range=ddt.sharding.ensemble_chunk(T, g, G))
             for g in range(G)]
    return O.ring_combine([p.ravel() for p in parts]).reshape(x.shape[0], nc)


def _device_lists():
    out = [[0, 0, 0]]
    try:
        import torch
        if torch.cuda.device_count() >= 2:
            out.append([0, 1])
    except Exception:
        pass
    return out


@pytest.mark.parametrize("devs", _device_lists(), ids=lambda d: "gpus" + "".join(map(str, d)))
def test_multi_device_handle_dealt_and_chunked(devs):
    """dte_create_multi: Dealt replicates the classed ensemble; Chunked keeps ring position r's contiguous tree range
    (boundaries that are not multiples of C, so chunks start mid-round) and ring-combines the [n][C] partials."""
    G = len(devs)
    nc, D, F, K, n = 3, 7, 64, 2, 5003
    T = 13 * G - 2                                      # chunks of 13 trees: 13 % 3 != 0
    W, FI = L.synth_ensemble(T, D, F, seed=3701)
    x = L.synth_tuples(0, n, F, seed=3702, missing_ppm=15000)
    wl, fl = L.pack_streams(W, FI, D)
    for mode in ("data", "ensemble"):
        regs = multi_node_regs(T, D, F, K, n, G, mode, batch_tuples=64)
        S = (regs[205] >> 36) & 0xFF
        want = (oracle_class_scores(W, FI, x, D, K, S, L.MISSING_DEFAULT, nc) if mode == "data"
                else _mc_ring_reference(W, FI, x, D, K, S, nc, G))
        with ddt.Engine(devs) as e:
            e.set_option(E.DTE_OPT_CHUNK_TUPLES, 700)      # several landing buffers, chunks that are not line-aligned x C
            write_regs(e, regs)
            e.load_ensemble(wl, fl, num_classes=nc)
            info = e.info()
            assert info["num_classes"] == nc and info["partition"] == (1 if mode == "data" else 2)
            for _ in range(2):
                sc, lb = e.infer_host(x)
                assert sc.shape == (n, nc)
                assert (sc.view(np.uint32) == want).all(), mode
                assert (lb == labels_of(want, nc)).all(), mode
            assert e.info()["tuples_out"] - info["tuples_out"] == 2 * n       # tuples, not score words


@pytest.mark.timeout(180)
@pytest.mark.parametrize("devs", [d for d in _device_lists() if len(set(d)) == len(d)], ids=lambda d: "gpus" + "".join(map(str, d)))
def test_multi_device_nccl_combine(devs):
    """DTE_OPT_COMBINE = 1 reduces n*C words with one ncclReduce: order free, so 1e-5 relative."""
    G = len(devs)
    nc, D, F, K, n = 3, 6, 64, 2, 20_011
    T = 13 * G - 2
    W, FI = L.synth_ensemble(T, D, F, seed=3801)
    x = L.synth_tuples(0, n, F, seed=3802, missing_ppm=15000)
    wl, fl = L.pack_streams(W, FI, D)
    regs = multi_node_regs(T, D, F, K, n, G, "ensemble")
    want = _mc_ring_reference(W, FI, x, D, K, (regs[205] >> 36) & 0xFF, nc, G)
    with ddt.Engine(devs) as e:
        e.set_option(E.DTE_OPT_COMBINE, 1)
        e.set_option(E.DTE_OPT_CHUNK_TUPLES, 4096)
        write_regs(e, regs)
        e.load_ensemble(wl, fl, num_classes=nc)
        sc, lb = e.infer_host(x)
        assert np.allclose(sc, want.view(np.float32), rtol=1e-5, atol=1e-7)
        assert (lb == labels_of(sc.view(np.uint32), nc)).all()


def test_two_engines_adjacent_chunks_ring_combined(torch_cuda):
    """Two single-device engines on one GPU hold adjacent tree chunks (the second starts at first_tree = 20, mid-round
    for C = 3); dte_ring_combine_device over n*C words + dte_class_labels_device gives the oracle ring."""
    torch = torch_cuda
    nc, T, D, F, K, n = 3, 41, 8, 64, 2, 3001
    W, FI = L.synth_ensemble(T, D, F, seed=3901)
    x = L.synth_tuples(0, n, F, seed=3902, missing_ppm=10000)
    wl, fl = L.pack_streams(W, FI, D)
    S = slots_for(21, nc, K)
    chunks = [(0, 20), (20, 21)]
    parts = [oracle_class_scores(W, FI, x, D, K, S, L.MISSING_DEFAULT, nc, tree_range=c) for c in chunks]
    want = O.ring_combine([p.ravel() for p in parts]).reshape(n, nc)
    dx = torch.from_numpy(x.view(np.int32)).cuda()
    st = torch.cuda.current_stream().cuda_stream
    bufs, engines = [], []
    for first, count in chunks:
        e = make_engine(T, D, F, K, S)
        e.load_ensemble(wl, fl, first_tree=first, num_local_trees=count, num_classes=nc)
        b = torch.empty((n, nc), dtype=torch.float32, device="cuda")
        e.infer_device(dx, n, b, None, stream=st)
        bufs.append(b)
        engines.append(e)
    torch.cuda.synchronize()
    for b, p in zip(bufs, parts):
        assert (b.cpu().numpy().view(np.uint32) == p).all()
    out = torch.empty((n, nc), dtype=torch.float32, device="cuda")
    lab = torch.empty(n, dtype=torch.uint8, device="cuda")
    engines[0].ring_combine_device(bufs, n * nc, out, None, stream=st)
    engines[0].class_labels_device(out, n, nc, lab, stream=st)
    torch.cuda.synchronize()
    assert (out.cpu().numpy().view(np.uint32) == want).all()
    assert (lab.cpu().numpy() == labels_of(want, nc)).all()
    for e in engines:
        e.close()


def test_refusals_and_info():
    T, D, F, K, n = 40, 5, 32, 2, 256
    W, FI = L.synth_ensemble(T, D, F, seed=4001)
    x = L.synth_tuples(0, n, F, seed=4002)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F, K, 1) as e:                # S*K*8 = 16 slots
        for bad in (0, 257):
            refused(lambda: e.load_ensemble(wl, fl, num_classes=bad), E.DTE_ERR_ARG)
        e.load_ensemble(wl, fl, num_classes=2)            # 20 trees per class > 16 slots
        assert e.info()["num_classes"] == 2
        refused(lambda: e.infer_host(x), E.DTE_ERR_CONFIG, "S >= 2")
        e.load_ensemble(wl, fl, num_classes=3)            # 14 / 13 / 13 trees fit 16 slots
        sc, lb = e.infer_host(x)
        assert sc.shape == (n, 3) and (sc.view(np.uint32) == oracle_class_scores(W, FI, x, D, K, 1, L.MISSING_DEFAULT, 3)).all()
        # a data-only line-stream run would reuse the resident 3-class ensemble: the result stream has one score per tuple
        e.softreg_write(201, 0x41 | ((F // 4) << 32))     # data_distributed | pcie_receiver_enabled, not host node
        refused(e.start, E.DTE_ERR_CONFIG)
        # a single-class load makes the same data-only run legal again
        e.load_ensemble(wl, fl)
        assert e.info()["num_classes"] == 1
        e.start()
        assert e.softreg_read(220) == 3                   # receiving data
    with make_engine(T, D, F, K, 1) as e:
        assert e.info()["num_classes"] == 0               # nothing resident
        lib = e._lib
        assert lib.dte_class_labels_device(e._h, None, 0, 0, None, None) == E.DTE_ERR_ARG
        assert lib.dte_class_labels_device(e._h, None, 0, 257, None, None) == E.DTE_ERR_ARG


def test_autotune_on_a_multiclass_ensemble():
    T, D, F, K, nc = 61, 12, 256, 8, 10
    W, FI = L.synth_ensemble(T, D, F, seed=4101)
    x = L.synth_tuples(0, 2000, F, seed=4102)
    S = slots_for(T, nc, K)
    wl, fl = L.pack_streams(W, FI, D)
    want = oracle_class_scores(W, FI, x, D, K, S, L.MISSING_DEFAULT, nc)
    with make_engine(T, D, F, K, S) as e:
        e.load_ensemble(wl, fl, num_classes=nc)
        rep = e.autotune(100_000)
        assert "chosen: dt_walk_tile<" in rep and "classes=10" in rep, rep
        sc, lb = e.infer_host(x)
        assert (sc.view(np.uint32) == want).all() and (lb == labels_of(want, nc)).all()
