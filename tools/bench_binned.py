"""Binned inference against the fp32 path on one H100: prints one JSON line.

Workloads: histogram-trained ensembles (every feature's thresholds snapped to 254 cuts, synth_ensemble(cuts=254)) in
bench.py's shapes: cfg3-hist (1024 trees, D = 12, F = 256, 50 M tuples resident), cfg2 (512 trees, D = 8, F = 128, 10 M)
and the cfg4 shard (1024 trees, D = 10, F = 256, 20 M); K = 8 as bench.py.  Per workload, with the paths alternated:
  * device-resident walks: dte_infer_device (fp32 tuples) against dte_infer_device_binned (u8 bins), median of --reps;
  * the binning kernel on its own (dte_bin_tuples_device);
  * host paths from pinned buffers: dte_infer_host (4F bytes per tuple) against dte_infer_host_binned (F bytes).
It checks that every score word of the binned walk equals the fp32 walk's, and a 4096-tuple sample against the oracle.
Card name and power limit are printed with the numbers.  bench.py is not involved.
    python tools/bench_binned.py [--reps 3] [--host-tuples 4000000] [--only cfg3_hist,cfg2,cfg4_shard]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import ddt_b200 as ddt  # noqa: E402
from oracle import oracle as O  # noqa: E402

L = ddt.layout
SEED = 0x7091E5
WORKLOADS = {"cfg3_hist": (1024, 12, 256, 50_000_000), "cfg2": (512, 8, 128, 10_000_000),
             "cfg4_shard": (1024, 10, 256, 20_000_000)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def run(tag, T, D, F, n, reps, n_host):
    K = 8
    W, FI = L.synth_ensemble(T, D, F, cuts=254)
    wl, fl = L.pack_streams(W, FI, D)
    e = ddt.Engine(0)
    e.configure(T, D, 4 * F, clusters=K, missing_value=L.MISSING_DEFAULT, n_tuples=n)
    e.load_ensemble(wl, fl, binned=True)
    st = torch.cuda.current_stream().cuda_stream
    x = torch.empty((n, F), dtype=torch.int32, device="cuda")
    e.synth_tuples_device(x, 0, n, F, SEED, 10000, L.MISSING_DEFAULT, stream=st)
    b = torch.empty((n, F), dtype=torch.uint8, device="cuda")
    s32 = torch.empty(n, dtype=torch.float32, device="cuda")
    s8 = torch.empty(n, dtype=torch.float32, device="cuda")
    e.bin_tuples_device(x, n, b, stream=st)                                    # warm-up of every kernel
    e.infer_device(x, n, s32, stream=st)
    e.infer_device_binned(b, n, s8, stream=st)
    torch.cuda.synchronize()
    walk32, walk8, binning = [], [], []
    for _ in range(reps):                                                       # paths alternated
        walk32.append(timed(lambda: e.infer_device(x, n, s32, stream=st)))
        walk8.append(timed(lambda: e.infer_device_binned(b, n, s8, stream=st)))
        binning.append(timed(lambda: e.bin_tuples_device(x, n, b, stream=st)))
    equal = bool(torch.equal(s32.view(torch.int32), s8.view(torch.int32)))
    # oracle sample: the synthetic tuples are regenerated bit for bit on the host
    idx = np.linspace(0, n - 4096, 4096 // 256, dtype=np.int64)
    xs = np.concatenate([L.synth_tuples(int(i), 256, F, seed=SEED) for i in idx])
    w_cls, f_cls = L.tree_cls(D)
    S = (T + 8 * K - 1) // (8 * K)
    want = O.scores(O.make_cfg(D, K, S, L.MISSING_DEFAULT, w_cls, f_cls, F // 4, T), wl, fl, xs, threads=O.max_threads())
    got = np.concatenate([s8[int(i):int(i) + 256].cpu().numpy().view(np.uint32) for i in idx])
    oracle_ok = int((got == want).sum())
    kname32, kname8 = e.kernel_name(), e.kernel_name_binned()
    nh = min(n, n_host)
    hx = e.host_alloc((nh, F), np.uint32)
    hx[:] = x[:nh].cpu().numpy().view(np.uint32)
    del x, s32, s8
    # host paths, pinned buffers of n_host tuples
    hb = e.host_alloc((nh, F), np.uint8)
    hs = e.host_alloc((nh,), np.float32)
    off, edges = e.bin_edges()
    hb[:] = b[:nh].cpu().numpy()
    del b
    torch.cuda.empty_cache()
    host32, host8 = [], []
    e.infer_host(hx, want_labels=False, out_scores=hs)
    ref = hs.copy()
    e.infer_host_binned(hb, want_labels=False, out_scores=hs)
    host_equal = bool((ref.view(np.uint32) == hs.view(np.uint32)).all())
    for _ in range(reps):
        t0 = time.perf_counter(); e.infer_host(hx, want_labels=False, out_scores=hs); host32.append(time.perf_counter() - t0)
        t0 = time.perf_counter(); e.infer_host_binned(hb, want_labels=False, out_scores=hs); host8.append(time.perf_counter() - t0)
    for a in (hx, hb, hs):
        e.host_free(a)
    e.close()
    med = lambda v: float(np.median(v))
    return {"workload": "%d trees, D=%d, %d features, 254 cuts per feature, %d tuples resident" % (T, D, F, n),
            "edges": int(len(edges)),
            "fp32_walk_Mtps": n / med(walk32) / 1e3, "binned_walk_Mtps": n / med(walk8) / 1e3,
            "binned_over_fp32": med(walk32) / med(walk8), "binning_kernel_Mtps": n / med(binning) / 1e3,
            "binning_kernel_GBps_in": n * F * 4 / med(binning) / 1e6,
            "fp32_walk_ms": walk32, "binned_walk_ms": walk8, "binning_ms": binning,
            "host_tuples": nh, "infer_host_pinned_Mtps": nh / med(host32) / 1e6, "infer_host_binned_pinned_Mtps": nh / med(host8) / 1e6,
            "all_score_words_equal": equal, "host_paths_equal": host_equal, "oracle_words_equal_of_4096": oracle_ok,
            "kernel_fp32": kname32, "kernel_binned": kname8}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-tuples", type=int, default=4_000_000)
    ap.add_argument("--only", default=",".join(WORKLOADS))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_binned needs the H100"
    name, power = card()
    out = {"card": name, "power_limit": power}
    for tag in args.only.split(","):
        out[tag] = run(tag, *WORKLOADS[tag], args.reps, args.host_tuples)
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
