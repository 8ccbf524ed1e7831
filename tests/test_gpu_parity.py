"""Parity tests proper: the CUDA path, called through the C ABI (libdte.so), against the oracle.

Bar: BIT-EXACT scores (raw fp32 words) and labels on one device — the kernels reproduce the
reference's summation order, so no tolerance is needed or used.  Every kernel variant is tested.
Nothing here reads the reference sources."""
import ctypes as C
import os

import numpy as np
import pytest

import ddt_b200 as ddt
from ddt_b200 import engine as E
from helpers import kat_arrays, oracle_cfg, make_engine, multi_node_regs as _multi_node_regs, refused, torch_cuda, L  # noqa: F401
from oracle import oracle as O

pytestmark = pytest.mark.gpu

VARIANTS = [E.DTE_KERNEL_GENERIC, E.DTE_KERNEL_TILE, E.DTE_KERNEL_TILE_STAGED, E.DTE_KERNEL_AUTO]


def run_engine_host(e, x, variant):
    e.set_kernel_variant(variant)
    sc, lb = e.infer_host(x)
    return sc.view(np.uint32), lb


def check_case(W, FI, x, D, K, S, missing=L.MISSING_DEFAULT, variants=VARIANTS, want=None):
    T, F = W.shape[0], x.shape[1]
    wl, fl = L.pack_streams(W, FI, D)
    if want is None:
        want = O.scores(oracle_cfg(D, K, S, missing, F, T), wl, fl, x, threads=8)
    want_lab = O.labels(want)
    with make_engine(T, D, F, K, S, missing) as e:
        e.load_ensemble(wl, fl)
        for v in variants:
            got, lab = run_engine_host(e, x, v)
            info = e.info()
            bad = np.nonzero(got != want)[0]
            assert bad.size == 0, "variant %s (ran %s): %d/%d scores differ, first at %d: got %08x want %08x" % (
                E.KERNEL_NAMES[v], E.KERNEL_NAMES[info["kernel_variant"]], bad.size, want.size, bad[0], got[bad[0]], want[bad[0]])
            assert (lab == want_lab).all()
    return want


# ---------------------------------------------------------------------------------------------
def test_kats_on_gpu(kats):
    for c in kats["cases"]:
        W, FI, x = kat_arrays(c)
        check_case(W, FI, x, c["D"], c["K"], c["S"], c["missing"], want=np.array(c["expect"], dtype=np.uint32))


def test_cfg1_baseline_config_bit_exact():
    # BASELINE cfg1: 16 trees, depth 4, 32 fp32 features, 10k tuples
    W, FI = L.synth_ensemble(16, 4, 32)
    x = L.synth_tuples(0, 10000, 32)
    want = check_case(W, FI, x, 4, 2, 1)
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "cfg1_scores_first64.npy"))
    assert (want[:64] == gold).all()


@pytest.mark.parametrize("D,T,F,K,S,n", [
    (1, 8, 4, 1, 1, 100), (2, 24, 8, 1, 3, 333), (3, 64, 16, 8, 1, 1000), (4, 16, 32, 1, 2, 4097),
    (5, 13, 64, 2, 1, 129), (6, 40, 64, 4, 2, 2000), (7, 100, 100, 4, 4, 1000), (8, 512, 128, 8, 8, 3000),
    (10, 64, 256, 2, 4, 1500), (12, 64, 256, 8, 1, 1000), (12, 24, 64, 1, 3, 600), (9, 17, 512, 1, 3, 300),
])
def test_random_ensembles_bit_exact(D, T, F, K, S, n):
    W, FI = L.synth_ensemble(T, D, F, seed=100 + D)
    x = L.synth_tuples(0, n, F, seed=200 + T, missing_ppm=20000)
    check_case(W, FI, x, D, K, S)


def test_adversarial_negative_operands():
    # thresholds and features in (-1,1): the int32 comparator differs from IEEE on both-negative pairs
    W, FI = L.synth_ensemble(64, 8, 64, seed=5, negative=True, bias=0.0)
    x = L.synth_tuples(0, 3000, 64, seed=6, missing_ppm=10000, signed=True)
    want = check_case(W, FI, x, 8, 8, 1)
    # sanity: an IEEE comparator would produce different scores on this set
    xf = x.view(np.float32)
    assert (xf < 0).mean() > 0.3


def test_wide_feature_indexes_use_the_wide_record():
    # feature indexes >= 512 select the 64-byte bottom record; F beyond the tile capacity falls back to generic
    for F, D, T in [(600, 6, 16), (1024, 5, 16), (2044, 4, 8)]:
        W, FI = L.synth_ensemble(T, D, F, seed=F)
        x = L.synth_tuples(0, 500, F, seed=F + 1)
        check_case(W, FI, x, D, 1, -(-T // 8))


def test_tuple_count_edge_cases():
    W, FI = L.synth_ensemble(16, 6, 32, seed=9)
    for n in (1, 31, 32, 33, 127, 128, 129, 4736, 4737):
        x = L.synth_tuples(0, n, 32, seed=n)
        check_case(W, FI, x, 6, 2, 1)
    with make_engine(16, 6, 32, 2, 1) as e:
        e.load_ensemble(*L.pack_streams(W, FI, 6))
        sc, lb = e.infer_host(np.zeros((0, 32), dtype=np.uint32))
        assert sc.size == 0 and lb.size == 0


def test_device_pointer_path_and_determinism(torch_cuda):
    torch = torch_cuda
    T, D, F, K, S, n = 128, 10, 256, 8, 2, 20000
    W, FI = L.synth_ensemble(T, D, F, seed=77)
    x = L.synth_tuples(0, n, F, seed=78)
    wl, fl = L.pack_streams(W, FI, D)
    want = O.scores(oracle_cfg(D, K, S, L.MISSING_DEFAULT, F, T), wl, fl, x, threads=8)
    with make_engine(T, D, F, K, S) as e:
        e.load_ensemble(wl, fl)
        dx = torch.from_numpy(x.view(np.int32)).cuda()
        ds = torch.empty(n, dtype=torch.float32, device="cuda")
        dl = torch.empty(n, dtype=torch.uint8, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        for v in VARIANTS:
            e.set_kernel_variant(v)
            ds.zero_()
            e.infer_device(dx, n, ds, dl, stream=st)
            torch.cuda.synchronize()
            got = ds.cpu().numpy().view(np.uint32)
            assert (got == want).all(), E.KERNEL_NAMES[v]
            assert (dl.cpu().numpy() == O.labels(want)).all()
        # permutation property: scores follow their tuples
        perm = torch.randperm(n, device="cuda")
        ds2 = torch.empty_like(ds)
        e.infer_device(dx[perm].contiguous(), n, ds2, None, stream=st)
        torch.cuda.synchronize()
        assert torch.equal(ds2.view(torch.int32), ds.view(torch.int32)[perm])
        assert e.info()["kernel_launches"] >= 5


def test_register_and_line_stream_interface():
    """Drive the engine exactly like a Catapult host: register writes, `start`, then ONE line stream
    (weights | feature indexes | tuples) in arbitrary chunks; read result lines back."""
    T, D, F, K, n = 16, 4, 32, 2, 1003
    W, FI = L.synth_ensemble(T, D, F, seed=21)
    x = L.synth_tuples(0, n, F, seed=22)
    wl, fl = L.pack_streams(W, FI, D)
    want = O.scores(oracle_cfg(D, K, 1, L.MISSING_DEFAULT, F, T), wl, fl, x).view(np.float32)
    stream = np.concatenate([wl.view(np.uint8).reshape(-1, 16), fl.view(np.uint8).reshape(-1, 16),
                             x.view(np.uint8).reshape(-1, 16)])
    with ddt.Engine(0) as e:
        regs = e.configure(T, D, 4 * F, clusters=K, n_tuples=n)
        assert e.softreg_read(220) == 0                       # receiver idle
        assert e.softreg_read(999) == 0xFFFFFFFFFFFFFFFF      # EngineCSR.sv:123
        with pytest.raises(E.DteError):
            e.stream_write(stream[:4])                         # not started
        e.start()
        assert e.softreg_read(220) == 1                       # RECEIVE_TREES
        rng = np.random.default_rng(0)
        pos, out = 0, []
        while pos < stream.shape[0]:
            take = int(rng.integers(1, 700))
            e.stream_write(stream[pos:pos + take])
            pos += take
            out.append(e.stream_read(97))
        out.append(e.stream_read(1 << 20))
        got = np.concatenate(out)
        assert e.softreg_read(221) == stream.shape[0]
        assert got.shape == (n // 4, 4)                       # the last 3 results never flush (ResultsCombiner.sv:153-155)
        assert (got.reshape(-1).view(np.uint32) == want[: (n // 4) * 4].view(np.uint32)).all()
        assert regs[207] & 0xFFFFFFFF == n // 4 and e.process_done()
        assert e.softreg_read(220) == 0                       # process_done -> the receiver is IDLE again (PCIeReceiver.sv:289-292)
        exec_ns = e.softreg_read(223)
        assert exec_ns > 0 and e.softreg_read(223) == exec_ns     # execCycles stops at process_done (DTInference.sv:330-345)
        assert e.softreg_read(222) > 0                        # progCycles: the tree stream took time
        with pytest.raises(E.DteError):
            e.stream_write(stream[:4])                         # idle until the next start
        # "load the model once, then any number of start + data runs": data-only restart
        e.softreg_write(201, (regs[201] & ~0x2) | 0x1)        # host_node=0, data_distributed=1
        e.start()
        assert e.softreg_read(220) == 3
        e.stream_write(x[:64].view(np.uint8).reshape(-1, 16))
        again = e.stream_read(100)
        assert (again.reshape(-1).view(np.uint32) == want[:64].view(np.uint32)).all()
        assert e.softreg_read(223) > 0 and e.info()["num_trees"] == T
        # appStatus[2] = {data_lines, prog_lines} (DTInference.sv:369): 64 tuples x 8 lines, no tree lines in this run
        assert e.softreg_read(123) == (64 * (F // 4)) << 32
        # appStatus[1] = {num_out_tuples, cluster_tree_res_out[0]}: K = 2 -> cluster 0 serves every 4th tuple, S = 1
        a1 = e.softreg_read(122)
        assert a1 >> 32 == 64 and (a1 & 0xFFFFFFFF) == -(-1003 * K // 8) + 64 * K // 8
        e.set_option(E.DTE_OPT_CYCLE_MHZ, 150)                # registers 222/223 as 150 MHz cycles
        ns_view = e.softreg_read(223)
        e.set_option(E.DTE_OPT_CYCLE_MHZ, 0)
        assert 0 < ns_view < e.softreg_read(223)
        # packet framing of the output stream: `last` every pcie_out_packet_numcls lines (reg 206[55:48] = 8)
        e.start()
        e.stream_write(x[:400].view(np.uint8).reshape(-1, 16))
        lines, last = e.stream_read_packets(37)
        lines2, last2 = e.stream_read_packets(1000)
        flags = np.concatenate([last, last2])
        assert flags.size == 100 and (np.nonzero(flags)[0] == np.arange(7, 100, 8)).all()
        assert (np.concatenate([lines, lines2]).reshape(-1).view(np.uint32) == want[:400].view(np.uint32)).all()


def test_error_paths():
    W, FI = L.synth_ensemble(8, 3, 16, seed=1)
    wl, fl = L.pack_streams(W, FI, 3)
    with ddt.Engine(0) as e:
        refused(lambda: e.load_ensemble(wl, fl), E.DTE_ERR_CONFIG)        # geometry registers not written yet
        e.configure(8, 3, 64, clusters=1)
        with pytest.raises(E.DteError):                       # no ensemble
            e.infer_host(np.zeros((4, 16), dtype=np.uint32))
        bad = FI.copy(); bad[0, 0] = 200                       # feature index beyond F
        refused(lambda: e.load_ensemble(*L.pack_streams(W, bad, 3)), E.DTE_ERR_UNSUPPORTED)
        early = FI.copy(); early[0, 0] |= 1 << 14              # early-leaf bit on the root: a one-level tree, legal
        early[0, 1:] = 200                                     # ... and everything below it is don't-care
        e.load_ensemble(*L.pack_streams(W, early, 3))
        with pytest.raises(E.DteError):                       # truncated index stream
            e.load_ensemble(wl, fl[:-1])
        e.load_ensemble(wl, fl)
        assert e.info()["num_trees"] == 8


def test_ensemble_chunks_ring_combine_matches_oracle(torch_cuda):
    """Ensemble-sharded semantics on one GPU: two engines hold the two contiguous chunks
    (PCIeReceiver.sv:241-264), partials are ring-added on the device (ResultsCombiner.sv:292-311)."""
    torch = torch_cuda
    T, D, F, K, n = 64, 6, 64, 2, 5000
    W, FI = L.synth_ensemble(T, D, F, seed=31)
    x = L.synth_tuples(0, n, F, seed=32)
    wl, fl = L.pack_streams(W, FI, D)
    dx = torch.from_numpy(x.view(np.int32)).cuda()
    st = torch.cuda.current_stream().cuda_stream
    parts, want_parts = [], []
    for g in range(2):
        first, count = ddt.sharding.ensemble_chunk(T, g, 2)
        Kd, Sd = ddt.sharding.shard_geometry(T, D, K, 2)
        e = make_engine(T, D, F, Kd, Sd)
        e.load_ensemble(wl, fl, first_tree=first, num_local_trees=count)
        p = torch.empty(n, dtype=torch.float32, device="cuda")
        e.infer_device(dx, n, p, None, stream=st)
        parts.append((e, p))
        cw, cf = L.pack_streams(W[first:first + count], FI[first:first + count], D)
        want_parts.append(O.scores(oracle_cfg(D, Kd, Sd, L.MISSING_DEFAULT, F, count), cw, cf, x, threads=8))
    torch.cuda.synchronize()
    for (e, p), wp in zip(parts, want_parts):
        assert (p.cpu().numpy().view(np.uint32) == wp).all()
    e0 = parts[0][0]
    tot = torch.empty(n, dtype=torch.float32, device="cuda")
    lab = torch.empty(n, dtype=torch.uint8, device="cuda")
    e0.ring_add_device(parts[1][1], parts[0][1], tot, n, stream=st)      # local + incoming
    e0.labels_device(tot, n, lab, stream=st)
    torch.cuda.synchronize()
    want = O.ring_combine(want_parts)
    assert (tot.cpu().numpy().view(np.uint32) == want).all()
    assert (lab.cpu().numpy() == O.labels(want)).all()
    for e, _ in parts:
        e.close()


def test_device_generator_matches_host_generator(torch_cuda):
    torch = torch_cuda
    F, n, first = 256, 3000, 123456789
    with ddt.Engine(0) as e:
        d = torch.empty((n, F), dtype=torch.int32, device="cuda")
        e.synth_tuples_device(d, first, n, F, 0x7091E5, 10000, L.MISSING_DEFAULT, stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        host = L.synth_tuples(first, n, F, seed=0x7091E5, missing_ppm=10000)
        assert (d.cpu().numpy().view(np.uint32) == host).all()


def test_full_size_config_properties(torch_cuda):
    """BASELINE cfg3 geometry (1024 trees, 12 levels, 256 features) at a size the oracle cannot
    sweep: size-independent properties + an oracle check of a sample."""
    torch = torch_cuda
    T, D, F, K = 1024, 12, 256, 8
    n = 400_000
    W, FI = L.synth_ensemble(T, D, F)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F, K, 16) as e:
        e.load_ensemble(wl, fl)
        st = torch.cuda.current_stream().cuda_stream
        dx = torch.empty((n, F), dtype=torch.int32, device="cuda")
        e.synth_tuples_device(dx, 0, n, F, 0x7091E5, 10000, L.MISSING_DEFAULT, stream=st)
        res = {}
        for v in (E.DTE_KERNEL_TILE, E.DTE_KERNEL_TILE_STAGED):
            e.set_kernel_variant(v)
            ds = torch.empty(n, dtype=torch.float32, device="cuda")
            e.infer_device(dx, n, ds, None, stream=st)
            torch.cuda.synchronize()
            res[v] = ds
        # (1) variants agree bit for bit on all 400k tuples
        assert torch.equal(res[E.DTE_KERNEL_TILE].view(torch.int32), res[E.DTE_KERNEL_TILE_STAGED].view(torch.int32))
        # (2) idempotence / determinism of a second launch
        ds2 = torch.empty(n, dtype=torch.float32, device="cuda")
        e.infer_device(dx, n, ds2, None, stream=st)
        torch.cuda.synchronize()
        assert torch.equal(ds2.view(torch.int32), res[E.DTE_KERNEL_TILE_STAGED].view(torch.int32))
        # (3) batch-split invariance: a window scored alone equals the same window of the big batch
        lo, hi = 100_003, 137_777
        dw = torch.empty(hi - lo, dtype=torch.float32, device="cuda")
        e.infer_device(dx[lo:hi], hi - lo, dw, None, stream=st)
        torch.cuda.synchronize()
        assert torch.equal(dw.view(torch.int32), ds2.view(torch.int32)[lo:hi])
        # (4) oracle on a sample: the first 512 and every 1000th tuple
        idx = np.unique(np.concatenate([np.arange(512), np.arange(0, n, 1000)]))
        xs = np.stack([L.synth_tuples(int(i), 1, F)[0] for i in idx])
        want = O.scores(oracle_cfg(D, K, 16, L.MISSING_DEFAULT, F, T), wl, fl, xs, threads=O.max_threads())
        got = ds2.cpu().numpy().view(np.uint32)[idx]
        assert (got == want).all()
        assert 0.02 < O.labels(want).mean() < 0.98          # both labels occur in the sample


def test_cpp_host_program_matches_python_path():
    """tools/dte_host.cpp: the C++ host with the profiler's parameter surface (N_trees, Depth_tree,
    Size_tuple_Bytes) drives the same engine through registers + line streams; its checksum must
    equal the oracle's on the identically generated ensemble and tuples."""
    import json
    import subprocess
    from ddt_b200 import build as B
    exe = B.build_host()
    T, D, F, K, n = 64, 6, 64, 8, 4000
    for mode in ("stream", "host"):
        out = subprocess.run([exe, str(T), str(D), str(4 * F), str(n), str(K), mode], capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stderr
        r = json.loads(out.stdout.strip().splitlines()[-1])
        W, FI = L.synth_ensemble(T, D, F)
        x = L.synth_tuples(0, n, F)
        wl, fl = L.pack_streams(W, FI, D)
        want = O.scores(oracle_cfg(D, K, 1, L.MISSING_DEFAULT, F, T), wl, fl, x, threads=8)
        assert r["results"] == n and r["score_words_sum"] == int(want.astype(np.uint64).sum()), (mode, r)


@pytest.mark.parametrize("mode", ["ensemble", "data"])
def test_multi_node_stream_partitioning(mode, torch_cuda):
    """N1: every 'device' (engine) replays the SAME line stream and keeps what PCIeReceiver would have
    sent it: tree chunks by numcls_local_weights/findexes (PCIeReceiver.sv:241-264) or data batches of
    core_data_batch_cls lines (:298-307)."""
    torch = torch_cuda
    T, D, F, K, n, ndev = 48, 5, 32, 2, 404, 3
    W, FI = L.synth_ensemble(T, D, F, seed=41)
    x = L.synth_tuples(0, n, F, seed=42)
    wl, fl = L.pack_streams(W, FI, D)
    stream = np.concatenate([wl.view(np.uint8).reshape(-1, 16), fl.view(np.uint8).reshape(-1, 16), x.view(np.uint8).reshape(-1, 16)])
    regs = _multi_node_regs(T, D, F, K, n, ndev, mode)
    outs = []
    for g in range(ndev):
        with ddt.Engine(0) as e:
            e.set_node(g)
            for a, v in sorted(regs.items()):
                e.softreg_write(a, v)
            e.start()
            for pos in range(0, stream.shape[0], 997):
                e.stream_write(stream[pos:pos + 997])
            outs.append(e.stream_read(1 << 20).reshape(-1).view(np.uint32).copy())
            assert e.info()["num_trees"] == (T // ndev if mode == "ensemble" else T)
    if mode == "ensemble":
        parts = []
        for g in range(ndev):
            first, count = ddt.sharding.ensemble_chunk(T, g, ndev)
            cw, cf = L.pack_streams(W[first:first + count], FI[first:first + count], D)
            S = -(-count // (8 * K))
            parts.append(O.scores(oracle_cfg(D, K, S, L.MISSING_DEFAULT, F, count), cw, cf, x))
        for g in range(ndev):
            assert (outs[g] == parts[g][: (n // 4) * 4]).all()
        # ring combine of the engines' partials on the device == the oracle's ring order
        with ddt.Engine(0) as e:
            acc = torch.from_numpy(outs[0].view(np.float32).copy()).cuda()
            for g in range(1, ndev):
                nxt = torch.from_numpy(outs[g].view(np.float32).copy()).cuda()
                e.ring_add_device(nxt, acc, acc, acc.numel(), stream=torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
            want = O.ring_combine([p[: (n // 4) * 4] for p in parts])
            assert (acc.cpu().numpy().view(np.uint32) == want).all()
    else:
        full = O.scores(oracle_cfg(D, K, -(-T // (8 * K)), L.MISSING_DEFAULT, F, T), wl, fl, x)
        deal = ddt.sharding.deal_batches(n * (F // 4), 2 * (F // 4), ndev)
        for g in range(ndev):
            idx = np.concatenate([np.arange(a // (F // 4), (a + c) // (F // 4)) for a, c in deal[g]])
            want = full[idx]
            assert (outs[g] == want[: (idx.size // 4) * 4]).all()


def test_randomised_geometry_stress():
    """40 random (D, T, F, K, S, n, missing pattern) draws, every kernel variant, raw feature words
    drawn from the FULL 32-bit space (NaN/Inf/negative/denormal patterns included — the comparator is
    an integer compare, DTPU.sv:655, so every pattern is in contract for features and thresholds)."""
    rng = np.random.default_rng(20260922)
    for it in range(40):
        D = int(rng.integers(1, 13))
        K = int(rng.choice([1, 2, 4, 8]))
        T = int(rng.integers(1, 70))
        S = max(1, -(-T // (8 * K)) + int(rng.integers(-1, 2)))          # sometimes one slot short / long
        F = 4 * int(rng.integers(1, 80))
        n = int(rng.integers(1, 700))
        W, FI = L.synth_ensemble(T, D, F, seed=int(rng.integers(1 << 40)))
        n_int = (1 << D) - 1
        # thresholds: arbitrary 32-bit words
        W[:, :n_int] = rng.integers(0, 1 << 32, size=(T, n_int), dtype=np.uint64).astype(np.uint32)
        x = rng.integers(0, 1 << 32, size=(n, F), dtype=np.uint64).astype(np.uint32)
        missing = int(rng.integers(0, 1 << 32))
        x[rng.random((n, F)) < 0.03] = missing
        # make some features exactly equal to thresholds (the 'not smaller -> right' edge)
        for _ in range(10):
            t, i = int(rng.integers(T)), int(rng.integers(n_int))
            x[int(rng.integers(n)), FI[t, i] & 0x7FF] = W[t, i]
        check_case(W, FI, x, D, K, S, missing=missing)


def test_deeper_than_rtl_limit():
    # the CSR field allows D up to 15; beyond 12 the staged ring no longer fits and the planner falls back
    D, T, F = 13, 8, 32
    W, FI = L.synth_ensemble(T, D, F, seed=13)
    x = L.synth_tuples(0, 300, F, seed=14)
    check_case(W, FI, x, D, 1, 1)


@pytest.mark.parametrize("tune", ["pair=1,ilp=8,stages=1", "pair=1,ilp=4,stages=2", "pair=2,stages=1", "pair=2,stages=2",
                                  "pair=4,stages=1", "pair=1,ilp=8,stages=2,warps=3", "pair=2,stages=1,warps=4",
                                  "pair=2,ilp=2,stages=2", "pair=2,stages=1,phased=1", "pair=1,ilp=8,stages=1,phased=1",
                                  "pair=4,stages=2,phased=1"])
def test_every_launch_plan_is_bit_exact(tune, monkeypatch):
    """The planner's alternatives (trees per warp x warps per tuple group x ring stages) must all give
    the oracle's words: DTE_TUNE pins a plan for engines created while it is set."""
    monkeypatch.setenv("DTE_TUNE", tune)
    T, D, F, K, S, n = 72, 9, 64, 4, 3, 1500          # T % 8 == 0 but 3 slots x 4 clusters x 8 = 96 > T: empty groups
    W, FI = L.synth_ensemble(T, D, F, seed=91)
    x = L.synth_tuples(0, n, F, seed=92, missing_ppm=20000)
    check_case(W, FI, x, D, K, S, variants=[E.DTE_KERNEL_TILE_STAGED, E.DTE_KERNEL_TILE])
    W, FI = L.synth_ensemble(16, 12, 256, seed=93)   # the headline geometry, few trees
    x = L.synth_tuples(0, 700, 256, seed=94)
    check_case(W, FI, x, 12, 8, 1, variants=[E.DTE_KERNEL_TILE_STAGED])


def test_fused_accumulate_epilogue(torch_cuda):
    """N3: the walk kernel adds its partial scores into a shared target with a system-scope reduction
    (dte_infer_device_accumulate).  Two contributors: a+b is commutative -> bit-exact with the ring;
    three contributors: the order is free -> 1e-5 relative (north_star tolerance), labels stable."""
    torch = torch_cuda
    T, D, F, K, n = 96, 7, 64, 2, 6000
    W, FI = L.synth_ensemble(T, D, F, seed=51)
    x = L.synth_tuples(0, n, F, seed=52)
    wl, fl = L.pack_streams(W, FI, D)
    dx = torch.from_numpy(x.view(np.int32)).cuda()
    st = torch.cuda.current_stream().cuda_stream
    for ndev in (2, 3):
        target = torch.zeros(n, dtype=torch.float32, device="cuda")
        parts, engines = [], []
        for g in range(ndev):
            first, count = ddt.sharding.ensemble_chunk(T, g, ndev)
            Kd, Sd = ddt.sharding.shard_geometry(T, D, K, ndev)
            e = make_engine(T, D, F, Kd, Sd)
            e.load_ensemble(wl, fl, first_tree=first, num_local_trees=count)
            e.infer_device_accumulate(dx, n, target, stream=st)
            engines.append(e)
            cw, cf = L.pack_streams(W[first:first + count], FI[first:first + count], D)
            parts.append(O.scores(oracle_cfg(D, Kd, Sd, L.MISSING_DEFAULT, F, count), cw, cf, x, threads=8))
        torch.cuda.synchronize()
        want = O.ring_combine(parts)
        got = target.cpu().numpy()
        if ndev == 2:
            assert (got.view(np.uint32) == want).all()
        else:
            assert np.allclose(got, want.view(np.float32), rtol=1e-5, atol=1e-7)
        assert (O.labels(got.view(np.uint32)) == O.labels(want)).mean() > 0.999
        for e in engines:
            e.close()


def test_shipped_plan_headline_geometry_multi_tile(capsys):
    """The kernel instantiation that ships for BASELINE cfg3 (D = 12, F = 256: 4 trees/warp x 2 warps/group, one
    64 KiB ring stage, phased refill), on enough tuples that every persistent CTA processes SEVERAL tiles (tile
    reload, ring wrap-around, step-parity exchange across tiles), bit-exact against the oracle.  This is the case
    tools/gpu_sanitize.sh runs under compute-sanitizer (racecheck / synccheck / memcheck), also with
    DTE_TUNE = pair=4 | ilp=8 | stages=2."""
    T, D, F, K, S = 24, 12, 256, 8, 1
    n = 160 * 132 * 2 + 77                               # 160 tuples per CTA, one CTA per SM on a 132-SM H100
    if os.environ.get("DTE_TEST_SANITIZER"):          # instrumented runs: 16 trees, CTAs 0..2 still process two tiles each
        T, n = 16, 160 * 132 + 333
    W, FI = L.synth_ensemble(T, D, F, seed=1201)
    x = L.synth_tuples(0, n, F, seed=1202, missing_ppm=15000)
    wl, fl = L.pack_streams(W, FI, D)
    want = O.scores(oracle_cfg(D, K, S, L.MISSING_DEFAULT, F, T), wl, fl, x, threads=O.max_threads())
    with make_engine(T, D, F, K, S) as e:
        e.load_ensemble(wl, fl)
        name = e.kernel_name()
        with capsys.disabled():
            print("\n[shipped-plan] DTE_TUNE=%r -> %s" % (os.environ.get("DTE_TUNE", ""), name))
        if not os.environ.get("DTE_TUNE"):
            assert name.startswith("dt_walk_tile<4, 2, 1, 0, 384>") and "phased=1" in name, name
        got, lab = run_engine_host(e, x, E.DTE_KERNEL_AUTO)
        assert e.info()["tuples_per_cta"] * e.info()["sm_count"] < n
    assert (got == want).all() and (lab == O.labels(want)).all()


def test_early_leaves_random_ensembles():
    """Bit 14 ("next node is leaf", DTPU.sv:596,661,712) with the build-defined rule (walk ends in the child's cell):
    random early leaves at random levels, garbage below them; every kernel variant equals the oracle."""
    rng = np.random.default_rng(14)
    for D, T, F in [(3, 8, 8), (6, 24, 32), (9, 16, 64), (12, 8, 256)]:
        W, FI = L.synth_ensemble(T, D, F, seed=1400 + D)
        n_int = (1 << D) - 1
        for t in range(T):
            for _ in range(int(rng.integers(0, 6))):
                lvl = int(rng.integers(0, D))
                i = (1 << lvl) - 1 + int(rng.integers(0, 1 << lvl))
                FI[t, i] |= 1 << 14
                # everything below node i's children is unreachable: fill with out-of-range indexes / noise
                lo, hi = 2 * (2 * i + 1) + 1, 2 * (2 * i + 2) + 2
                while lo < n_int:
                    FI[t, lo:min(hi, n_int - 1) + 1] = 0x7FF
                    lo, hi = 2 * lo + 1, 2 * hi + 2
        x = L.synth_tuples(0, 777, F, seed=1500 + D, missing_ppm=20000)
        check_case(W, FI, x, D, 2, -(-T // 16))


def test_autotune_picks_a_plan_and_stays_bit_exact():
    """dte_autotune times the planner's alternatives on the resident ensemble and pins the fastest; whatever it picks,
    scores stay the oracle's words (VERDICT r1 weak item 13: the built-in plan choice is a fitted heuristic)."""
    for T, D, F in [(64, 9, 64), (32, 12, 256), (40, 7, 512)]:
        W, FI = L.synth_ensemble(T, D, F, seed=700 + D)
        x = L.synth_tuples(0, 3000, F, seed=701 + D)
        wl, fl = L.pack_streams(W, FI, D)
        want = O.scores(oracle_cfg(D, 8, -(-T // 64), L.MISSING_DEFAULT, F, T), wl, fl, x, threads=8)
        with make_engine(T, D, F, 8, -(-T // 64)) as e:
            e.load_ensemble(wl, fl)
            before = e.kernel_name()
            rep = e.autotune(200_000)
            assert "chosen: dt_walk_tile<" in rep and rep.count("M tuples/s") >= 3, rep
            assert e.kernel_name() in rep
            got, lab = run_engine_host(e, x, E.DTE_KERNEL_AUTO)
            assert (got == want).all() and (lab == O.labels(want)).all(), (before, rep)
