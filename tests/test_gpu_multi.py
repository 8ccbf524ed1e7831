"""One handle, several devices (dte_create_multi): the whole ring behind the host node's register file and line
streams — SURVEY 8(e) / VERDICT NS1.  Parametrised over [0, 0, 0] (three ring positions sharing one GPU: runs on a
one-GPU box and exercises every host-side path), and over real device lists when the box has them.
Bar: bit-exact with the oracle, in GLOBAL tuple order; the ensemble-sharded combine is the reference's RING order
(ResultsCombiner.sv:292-311,359-368), so it is bit-exact too — scores and labels."""
import numpy as np
import pytest

import ddt_b200 as ddt
from ddt_b200 import engine as E
from helpers import oracle_cfg, multi_node_regs, L
from oracle import oracle as O

pytestmark = pytest.mark.gpu


def _device_lists():
    out = [[0, 0, 0]]
    try:
        import torch
        n = torch.cuda.device_count()
    except Exception:
        n = 0
    if n >= 2:
        out.append([0, 1])
    if n >= 4:
        out.append([3, 1, 0, 2])
    if n >= 8:
        out.append(list(range(8)))
    return out


DEVICE_LISTS = _device_lists()


def _case(T, D, F, n, seed):
    W, FI = L.synth_ensemble(T, D, F, seed=seed)
    x = L.synth_tuples(0, n, F, seed=seed + 1, missing_ppm=15000)
    wl, fl = L.pack_streams(W, FI, D)
    stream = np.concatenate([wl.view(np.uint8).reshape(-1, 16), fl.view(np.uint8).reshape(-1, 16), x.view(np.uint8).reshape(-1, 16)])
    return W, FI, x, wl, fl, stream


def _ensemble_reference(W, FI, x, D, K, ndev):
    """Oracle: per-chunk partial scores, ring-combined host first."""
    T, F = W.shape[0], x.shape[1]
    parts = []
    for g in range(ndev):
        first, count = ddt.sharding.ensemble_chunk(T, g, ndev)
        cw, cf = L.pack_streams(W[first:first + count], FI[first:first + count], D)
        S = -(-(-(-T // ndev)) // (8 * K))
        parts.append(O.scores(oracle_cfg(D, K, S, L.MISSING_DEFAULT, F, count), cw, cf, x, threads=8))
    return O.ring_combine(parts), parts


def _write_regs(e, regs):
    for a, v in sorted(regs.items()):
        e.softreg_write(a, v)


@pytest.mark.parametrize("devs", DEVICE_LISTS, ids=lambda d: "gpus" + "".join(map(str, d)))
def test_data_sharded_line_stream_global_order(devs):
    """broadcast_trees=1, data dealt in batches of core_data_batch_cls lines (PCIeReceiver.sv:298-307): ONE stream in,
    ONE result stream out, in global tuple order, bit-exact with the single-device oracle."""
    G = len(devs)
    T, D, F, K, n = 40, 6, 64, 2, 2407
    W, FI, x, wl, fl, stream = _case(T, D, F, n, 61)
    want = O.scores(oracle_cfg(D, K, -(-T // (8 * K)), L.MISSING_DEFAULT, F, T), wl, fl, x, threads=8)
    for batch_tuples in (2, 128):
        regs = multi_node_regs(T, D, F, K, n, G, "data", batch_tuples=batch_tuples)
        with ddt.Engine(devs) as e:
            _write_regs(e, regs)
            e.start()
            got, pos = [], 0
            rng = np.random.default_rng(batch_tuples)
            while pos < stream.shape[0]:
                take = int(rng.integers(1, 3000))
                e.stream_write(stream[pos:pos + take])
                pos += take
                if rng.random() < 0.3:
                    got.append(e.stream_read(int(rng.integers(1, 200))))
            got.append(e.stream_read(1 << 20))
            out = np.concatenate(got).reshape(-1).view(np.uint32)
            info = e.info()
            assert info["num_devices"] == G and info["partition"] == 1 and info["num_trees"] == T
            assert out.size == (n // 4) * 4 and (out == want[: out.size]).all()
            assert e.process_done()
            assert e.softreg_read(224) > 0                      # lines left for the other ring positions


@pytest.mark.parametrize("devs", DEVICE_LISTS, ids=lambda d: "gpus" + "".join(map(str, d)))
def test_ensemble_sharded_line_stream_ring_exact(devs):
    """broadcast_data=1, aggreg_enabled=1: tree chunks by numcls_local_weights/findexes (PCIeReceiver.sv:241-264), the
    tuples broadcast (InputDistributor.sv:199-204), partials combined in RING order by one kernel — raw words equal."""
    G = len(devs)
    T, D, F, K, n = 24 * G, 5, 32, 2, 1811
    W, FI, x, wl, fl, stream = _case(T, D, F, n, 71)
    want, parts = _ensemble_reference(W, FI, x, D, K, G)
    regs = multi_node_regs(T, D, F, K, n, G, "ensemble")
    with ddt.Engine(devs) as e:
        e.set_option(E.DTE_OPT_CHUNK_TUPLES, 512)               # several landing buffers -> slot reuse, partial flushes
        _write_regs(e, regs)
        e.start()
        for pos in range(0, stream.shape[0], 1777):
            e.stream_write(stream[pos:pos + 1777])
        out = e.stream_read(1 << 20).reshape(-1).view(np.uint32)
        info = e.info()
        assert info["partition"] == 2 and info["num_trees"] == T
        assert out.size == (n // 4) * 4 and (out == want[: out.size]).all()
        # host fast path on the same handle: scores AND labels, all n tuples (no line flush rule here)
        sc, lb = e.infer_host(x)
        assert (sc.view(np.uint32) == want).all() and (lb == O.labels(want)).all()
        # a permuted devices_list (registers 208-210): ring position i served by device ID list[i]; same answer,
        # and the resident chunks may not be reused under another ring order
        perm = [int(v) for v in np.random.default_rng(G).permutation(G)]
        if perm == list(range(G)):
            perm = perm[1:] + perm[:1]
        r208 = 0
        for i, d in enumerate(perm):
            r208 |= d << (8 * i)
        e.softreg_write(208, r208)
        with pytest.raises(E.DteError) as ei:
            e.infer_host(x)
        assert ei.value.code == -3
        e.start()
        e.stream_write(stream)
        out2 = e.stream_read(1 << 20).reshape(-1).view(np.uint32)
        assert (out2 == want[: out2.size]).all()
        sc, _ = e.infer_host(x)
        assert (sc.view(np.uint32) == want).all()


@pytest.mark.parametrize("devs", DEVICE_LISTS, ids=lambda d: "gpus" + "".join(map(str, d)))
def test_multi_fast_paths_load_and_infer_host(devs):
    """dte_load_ensemble + dte_infer_host on a multi-device handle: reg 201 picks the partition."""
    G = len(devs)
    T, D, F, K, n = 16 * G, 7, 64, 4, 5003
    W, FI, x, wl, fl, _ = _case(T, D, F, n, 81)
    full = O.scores(oracle_cfg(D, K, -(-T // (8 * K)), L.MISSING_DEFAULT, F, T), wl, fl, x, threads=8)
    ring, _ = _ensemble_reference(W, FI, x, D, K, G)
    for mode, want in (("data", full), ("ensemble", ring)):
        with ddt.Engine(devs) as e:
            e.set_option(E.DTE_OPT_CHUNK_TUPLES, 700)
            _write_regs(e, multi_node_regs(T, D, F, K, n, G, mode, batch_tuples=64))
            e.load_ensemble(wl, fl)
            for _ in range(2):
                sc, lb = e.infer_host(x)
                assert (sc.view(np.uint32) == want).all(), mode
                assert (lb == O.labels(want)).all()
            assert e.info()["kernel_launches"] >= 2 * G
            with pytest.raises(E.DteError) as ei:              # device pointers belong to one device
                e.infer_device(0x1000, 4, 0x2000)
            assert ei.value.code == -4


def _dealt_tuples(n, bt, G, pos):
    """Tuples ring position `pos` keeps when n tuples are dealt in batches of bt tuples over G positions, round-robin
    from position 0 (PCIeReceiver.sv:298-307): full batches first, then the short last batch (if any)."""
    full, rem = divmod(n, bt)
    return (full // G + (1 if pos < full % G else 0)) * bt + (rem if full % G == pos else 0)


def _pair(hi, lo):
    return ((hi & 0xFFFFFFFF) << 32) | (lo & 0xFFFFFFFF)


STATUS_CASES = [("whole", 0), ("own_batches", 0)] + [(p, d) for p in ("dealt", "chunked") for d in DEVICE_LISTS]


@pytest.mark.parametrize("partition,devs", STATUS_CASES,
                         ids=lambda v: v if isinstance(v, str) else "gpus" + "".join(map(str, v if isinstance(v, list) else [v])))
def test_status_registers_and_info_per_partition(partition, devs):
    """One line-stream job in each of the four partitions of a handle; the status registers 121-126 / 220 / 224-226
    and the info() counters, each written as arithmetic on the job's parameters (DTInference.sv:367-372).
      whole        single device, keeps every tuple
      own_batches  single device standing for ring position 1 (dte_set_node) on a dealt stream: keeps its batches
      dealt        multi-device, trees replicated, data dealt in batches over the ring
      chunked      multi-device, trees cut in per-device chunks, data broadcast, partials ring-combined"""
    G = len(devs) if isinstance(devs, list) else 3          # ring positions (numDevs, reg 203[39:32])
    T, D, F, K, n, bt = 48, 6, 64, 2, 132, 8                 # 132 = 16 full batches of 8 tuples + a short batch of 4
    assert T % G == 0 and n % 4 == 0 and bt % 4 == 0        # whole chunks, whole result lines
    tl = F // 4                                              # lines per tuple (tuple_numcls)
    w_cls, f_cls = L.tree_cls(D)
    tree_lines = T * (w_cls + f_cls)
    per = T // G                                             # trees per ring position when chunked
    _, _, x, wl, fl, stream = _case(T, D, F, n, 151)
    single = partition in ("whole", "own_batches")
    if partition == "whole":
        regs = E.csr_from_profile(T, D, 4 * F, K, L.MISSING_DEFAULT, n)
    else:
        regs = multi_node_regs(T, D, F, K, n, G, "ensemble" if partition == "chunked" else "data", batch_tuples=bt)
    S = -(-(per if partition == "chunked" else T) // (8 * K))
    n0 = n if partition in ("whole", "chunked") else _dealt_tuples(n, bt, G, 0)
    mine = _dealt_tuples(n, bt, G, 1) if partition == "own_batches" else n    # results this handle exposes
    if partition == "own_batches":                           # process_done counts this node's own result lines
        regs[207] = (regs[207] & ~0xFFFFFFFF) | (mine // 4)
    # ring position 0's tuples drive the cluster-0 counters; on a own_batches handle that is this node's device
    nt = mine if partition == "own_batches" else n0
    c0 = -(-nt * K // 8)                                     # tuple i uses clusters (i*K)%8 .. +K-1
    prog_local = per * (w_cls + f_cls) if partition == "chunked" else tree_lines
    sent = {"whole": 0,                                      # lines that left for other ring positions
            "own_batches": (n - n0) * tl,
            "dealt": tree_lines + (n - n0) * tl,
            "chunked": tree_lines - prog_local + n * tl}[partition]
    res_lines = {"whole": 0, "own_batches": 0, "dealt": (n - n0) // 4, "chunked": n // 4}[partition]
    pk = 8                                                   # data_packet_numcls of csr_from_profile (reg 206[31:24])

    def check(state, nt_now, c0_now, cum, res):
        r = {a: e.softreg_read(a) for a in (220, 121, 122, 123, 124, 125, 126, 224, 225, 226)}
        assert r == {220: state, 121: _pair(c0_now, cum + c0_now), 122: _pair(nt_now, (cum + c0_now) * S),
                     123: _pair(nt_now * tl, prog_local), 124: _pair(nt_now, cum + c0_now), 125: _pair(cum + c0_now, res),
                     126: _pair(cum + c0_now, (cum + c0_now) * tl), 224: sent, 225: -(-sent // pk), 226: sent}, partition

    with ddt.Engine(devs) as e:
        e.set_option(E.DTE_OPT_CHUNK_TUPLES, 16)             # several landing buffers per device
        if partition == "own_batches":
            e.set_node(1)
        _write_regs(e, regs)
        e.start()
        for pos in range(0, stream.shape[0], 997):
            e.stream_write(stream[pos:pos + 997])
        check(3, nt, c0, 0, 0)                               # RECEIVE_DATA, nothing read yet
        out = e.stream_read(1 << 20)
        assert out.shape[0] == mine // 4
        assert e.process_done()
        check(0, 0, 0, c0, res_lines)                        # IDLE; cluster counters rolled into the cumulative ones
        info = e.info()
        assert {k: info[k] for k in ("partition", "num_trees", "num_devices", "tuples_in", "tuples_out")} == {
            "partition": {"whole": 0, "own_batches": 0, "dealt": 1, "chunked": 2}[partition], "num_trees": T,
            "num_devices": 1 if single else G, "tuples_in": n, "tuples_out": mine}
        # a second run that is restarted before it completes: `start` rolls its cluster counters over as well
        e.start()
        e.stream_write(stream)
        e.start()
        assert e.softreg_read(220) == 1                      # RECEIVE_TREES
        assert e.softreg_read(121) == _pair(0, 2 * c0) and e.softreg_read(126) == _pair(2 * c0, 2 * c0 * tl)


def test_multi_handle_refuses_unsupported_partitions():
    T, D, F, K = 16, 4, 32, 2
    with ddt.Engine([0, 0]) as e:
        e.configure(T, D, 4 * F, clusters=K)                    # single-device flags on a 2-device handle
        with pytest.raises(E.DteError) as ei:
            e.start()
        assert ei.value.code == -3
        regs = multi_node_regs(T, D, F, K, 64, 2, "ensemble")
        regs[201] &= ~0x10                                      # tree chunks + broadcast data but NO aggregate
        _write_regs(e, regs)
        with pytest.raises(E.DteError):
            e.start()
        regs = multi_node_regs(T, D, F, K, 64, 3, "data")       # numDevs = 3 on a 2-device handle
        _write_regs(e, regs)
        with pytest.raises(E.DteError):
            e.start()
        regs = multi_node_regs(T, D, F, K, 64, 2, "ensemble")
        regs[208] = 0x0101                                      # devices_list is not a permutation
        _write_regs(e, regs)
        with pytest.raises(E.DteError):
            e.start()
        with pytest.raises(E.DteError):
            e.set_node(1)


def test_result_queue_back_pressure_and_restart_geometry_check():
    T, D, F, K, n = 16, 4, 32, 2, 400
    W, FI, x, wl, fl, stream = _case(T, D, F, n, 91)
    want = O.scores(oracle_cfg(D, K, 1, L.MISSING_DEFAULT, F, T), wl, fl, x)
    with ddt.Engine(0) as e:
        e.set_option(E.DTE_OPT_RESULT_QUEUE_LINES, 16)          # 64 results
        regs = e.configure(T, D, 4 * F, clusters=K, n_tuples=n)
        e.start()
        e.stream_write(stream[: wl.shape[0] + fl.shape[0]])
        lines = x.view(np.uint8).reshape(-1, 16)
        tl = F // 4
        e.stream_write(lines[: 60 * tl])
        with pytest.raises(E.DteError) as ei:                   # pcie_full_out: nothing is consumed
            e.stream_write(lines[60 * tl: 70 * tl])
        assert ei.value.code == E.DTE_ERR_BACKPRESSURE
        got = [e.stream_read(1 << 10)]
        assert got[0].shape[0] == 15
        for lo in range(60, n, 50):                             # read as we go: the bounded queue never overflows
            e.stream_write(lines[lo * tl: min(n, lo + 50) * tl])
            got.append(e.stream_read(1 << 10))
        out = np.concatenate(got).reshape(-1).view(np.uint32)
        assert (out == want).all()
        # a data-only restart whose registers disagree with the resident ensemble is refused (tuple_numcls 8 -> 4)
        r204 = (regs[204] & ~(0xFFFF << 48)) | ((F // 8) << 48)
        e.softreg_write(204, r204)
        e.softreg_write(201, (regs[201] & ~0x2) | 0x1)
        with pytest.raises(E.DteError) as ei:
            e.start()
        assert ei.value.code == -3
        with pytest.raises(E.DteError):
            e.infer_host(x[:, : F // 2].copy())
        e.softreg_write(204, regs[204])
        e.start()
        e.stream_write(lines[: 8 * tl])
        assert (e.stream_read(10).reshape(-1).view(np.uint32) == want[:8]).all()
        # a failed load leaves the resident ensemble and its geometry in place
        bad = FI.copy(); bad[0, 0] = 40                        # feature index >= F
        with pytest.raises(E.DteError):
            e.load_ensemble(*L.pack_streams(W, bad, D))
        sc, _ = e.infer_host(x[:16])
        assert (sc.view(np.uint32) == want[:16]).all()


def test_ring_combine_kernel_against_oracle_ring():
    """dte_ring_combine_device: G partial vectors -> ((p0+p1)+p2)+... with add.rn.ftz.f32, n % 4 != 0 tail, labels."""
    import torch
    rng = np.random.default_rng(5)
    n = 100_003
    for G in (1, 2, 3, 8, 20):
        parts = []
        for g in range(G):
            v = (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4, n)).astype(np.float32)
            v[rng.random(n) < 0.01] = 0.0
            parts.append(v)
        if G >= 2:
            parts[1][:1000] = -parts[0][:1000]                  # exact cancellation -> +0
            parts[1][1000:2000] = np.nextafter(-parts[0][1000:2000], np.float32(0))   # results below the normal range flush
        want = O.ring_combine([p.view(np.uint32) for p in parts])
        d = [torch.from_numpy(p).cuda() for p in parts]
        out = torch.empty(n, dtype=torch.float32, device="cuda")
        lab = torch.empty(n + 3, dtype=torch.uint8, device="cuda")
        with ddt.Engine(0) as e:
            e.ring_combine_device(d, n, out, lab, stream=torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
        assert (out.cpu().numpy().view(np.uint32) == want).all(), G
        assert (lab[:n].cpu().numpy() == O.labels(want)).all()


def test_default_stream_handle_orders_with_torch_work():
    """ADVICE r1: torch's default-stream handle is 0; the wrapper passes cudaStreamLegacy so the walk is ordered with
    the caller's default-stream work (here: the tuples are produced on that stream right before the call)."""
    import torch
    T, D, F, K, n = 64, 8, 64, 8, 50_000
    W, FI, x, wl, fl, _ = _case(T, D, F, n, 95)
    want = O.scores(oracle_cfg(D, K, 1, L.MISSING_DEFAULT, F, T), wl, fl, x, threads=8)
    hx = torch.from_numpy(x.view(np.int32)).pin_memory()
    with ddt.Engine(0) as e:
        e.configure(T, D, 4 * F, clusters=K)
        e.load_ensemble(wl, fl)
        ds = torch.empty(n, dtype=torch.float32, device="cuda")
        for _ in range(3):
            dx = torch.zeros((n, F), dtype=torch.int32, device="cuda")
            big = torch.empty(64 << 20, dtype=torch.uint8, device="cuda").zero_()     # keep the default stream busy
            dx.copy_(hx, non_blocking=True)                                            # producer on the default stream
            e.infer_device(dx, n, ds, None, stream=torch.cuda.current_stream().cuda_stream)   # == 0
            got = ds.cpu().numpy().view(np.uint32)                                     # consumer on the default stream
            assert (got == want).all()
            del big


@pytest.mark.parametrize("devs", DEVICE_LISTS, ids=lambda d: "gpus" + "".join(map(str, d)))
def test_cpp_host_drives_the_whole_ring(devs):
    """tools/dte_host.cpp over dte_create_multi: the C++ host (profiler-style parameters) runs both partitions on every GPU
    of the list through registers + ONE line stream, and through the host fast path; checksums against the oracle."""
    import json
    import subprocess
    from ddt_b200 import build as B
    exe = B.build_host()
    G = len(devs)
    T, D, F, K, n = 16 * G, 6, 64, 4, 6000
    W, FI = L.synth_ensemble(T, D, F)
    x = L.synth_tuples(0, n, F)
    wl, fl = L.pack_streams(W, FI, D)
    full = O.scores(oracle_cfg(D, K, -(-T // (8 * K)), L.MISSING_DEFAULT, F, T), wl, fl, x, threads=8)
    ring, _ = _ensemble_reference(W, FI, x, D, K, G)
    for part, want in (("data", full), ("ensemble", ring)):
        for mode in ("stream", "host"):
            out = subprocess.run([exe, str(T), str(D), str(4 * F), str(n), str(K), mode, ",".join(map(str, devs)), part],
                                 capture_output=True, text=True, timeout=600)
            assert out.returncode == 0, out.stderr
            r = json.loads(out.stdout.strip().splitlines()[-1])
            assert r["gpus"] == G and r["partition"] == part
            assert r["results"] == n and r["score_words_sum"] == int(want.astype(np.uint64).sum()), (part, mode, r)


@pytest.mark.timeout(180)
@pytest.mark.parametrize("devs", [d for d in DEVICE_LISTS if len(set(d)) == len(d)], ids=lambda d: "gpus" + "".join(map(str, d)))
def test_nccl_combine_option(devs):
    """DTE_OPT_COMBINE = 1: the partial scores are summed by ONE ncclReduce (libnccl dlopen'ed by libdte.so) instead of
    the ring-order kernel — north_star's wording; the order is NCCL's, so 1e-5 relative (2 devices: a + b is commutative,
    still bit-exact), labels stable."""
    G = len(devs)
    T, D, F, K, n = 16 * G, 6, 64, 2, 20_011
    W, FI, x, wl, fl, _ = _case(T, D, F, n, 131)
    want, _ = _ensemble_reference(W, FI, x, D, K, G)
    with ddt.Engine(devs) as e:
        e.set_option(E.DTE_OPT_COMBINE, 1)
        e.set_option(E.DTE_OPT_CHUNK_TUPLES, 4096)
        _write_regs(e, multi_node_regs(T, D, F, K, n, G, "ensemble"))
        e.load_ensemble(wl, fl)
        sc, lb = e.infer_host(x)
        if G == 2:
            assert (sc.view(np.uint32) == want).all()
        else:
            assert np.allclose(sc, want.view(np.float32), rtol=1e-5, atol=1e-7)
        assert (lb == O.labels(sc.view(np.uint32))).all()
        assert (lb == O.labels(want)).mean() > 0.999
        e.set_option(E.DTE_OPT_COMBINE, 0)                      # back to the ring kernel on the same handle: bit-exact
        sc2, lb2 = e.infer_host(x)
        assert (sc2.view(np.uint32) == want).all() and (lb2 == O.labels(want)).all()
