"""Approximate (Saabas) contributions against the leaf and score walks on one H100: prints one JSON line.

Workloads: bench.py's ensembles and tuple seeds (K = 8) with layout.synth_covers: cfg2 (512 trees, D = 8, F = 128), the
cfg4 shard (1024 trees, D = 10, F = 256, ensemble seed 0xE5E) and cfg3 (1024 trees, D = 12, F = 256).  Per workload, on
one handle loaded with dte_load_ensemble_approx_contribs, over the same device-resident synthetic tuples (--tuples, 2 M
by default; the output takes 4 (F + 1) bytes per tuple): dte_infer_device_approx_contribs, dte_infer_device_leaves (the
kernel and plan of pass 1, into a [n][T] buffer of its own) and dte_infer_device (the score walk), alternated round by
round, median of --reps rounds after one warm-up round, each timed with CUDA events around the call.

Pass split: a separate run under torch.profiler (CUDA activities) sums the device time of each kernel of one approx call:
pass 1 (dt_walk_*_leaf) and pass 2 (dt_approx_generic).  Profiling is kept out of the timed rounds.

Pass-2 model per tuple, from the shapes (complete trees, so every path has D steps; Tu = trees the run adds):
  fp64 additions: Tu (D + 1); table loads: Tu (D (8 + 2) + 8) bytes (delta, feature, E[root]); accumulator traffic:
  Tu (D + 1) 16 bytes (load and store of an fp64 word) plus (F + 1) 20 bytes (zero it, read it back, write the fp32
  word); cells: 2 Tu bytes.

Checks on every run: efficiency on every tuple (sum_f phi + bias against the same handle's score word, within
U sum|phi| + (T + 1) U sum_t max|leaf_t|, U = 2^-24) and word equality of --sample tuples with
tests/approx_ref.approx_contribs.  The TreeSHAP rate beside it is README's (dte_infer_device_contribs, same workloads).
    python tools/bench_approx_contribs.py [--reps 3] [--sample 64] [--tuples N] [--only cfg2,cfg4_shard,cfg3] [--out F]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import ddt_b200 as ddt  # noqa: E402
from approx_ref import approx_contribs  # noqa: E402

L = ddt.layout
SEED = 0x7091E5
MISSING_PPM = 10000
K = 8
U = 2.0 ** -24
WORKLOADS = {"cfg2": (512, 8, 128, None), "cfg4_shard": (1024, 10, 256, 0xE5E), "cfg3": (1024, 12, 256, None)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in out.split(",")]
    except Exception:
        return [torch.cuda.get_device_name(0), "unknown", "unknown", "unknown"]


def progress(*a):
    print(*a, file=sys.stderr, flush=True)


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def pass_split(fn):
    """Device ms of pass 1 and pass 2 of one call, from torch.profiler's kernel records."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    p1 = p2 = 0.0
    for ev in prof.events():
        us = getattr(ev, "device_time", 0.0) or 0.0
        if "dt_approx_generic" in ev.name:
            p2 += us
        elif "_leaf" in ev.name and "dt_walk" in ev.name:
            p1 += us
    return p1 * 1e-3, p2 * 1e-3


def run(tag, reps, sample, n):
    T, D, F, seed = WORKLOADS[tag]
    W, FI = L.synth_ensemble(T, D, F) if seed is None else L.synth_ensemble(T, D, F, seed=seed)
    cov = L.synth_covers(FI, D)
    wl, fl = L.pack_streams(W, FI, D)
    e = ddt.Engine(0)
    e.configure(T, D, 4 * F, clusters=K)
    e.load_ensemble(wl, fl, covers=cov, approx=True)
    info = e.info()
    Tu = min(T, 8 * K * max(1, -(-T // (8 * K))))
    dx = torch.empty((n, F), dtype=torch.float32, device="cuda")
    e.synth_tuples_device(dx, 0, n, F, SEED, MISSING_PPM, L.MISSING_DEFAULT)
    out = torch.empty((n, F + 1), dtype=torch.float32, device="cuda")
    leaves = torch.empty((n, T), dtype=torch.int16, device="cuda")
    sc = torch.empty(n, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    res = {"trees": T, "D": D, "F": F, "tuples": n, "kernels": e.kernel_name_approx_contribs(),
           "leaf_kernel": e.kernel_name_leaves(), "ensemble_bytes": int(info["ensemble_bytes"])}
    progress("%s: %d tuples, %s" % (tag, n, res["kernels"]))
    calls = {"approx": lambda: e.infer_device_approx_contribs(dx, n, out),
             "leaf_walk": lambda: e.infer_device_leaves(dx, n, leaves),
             "score_walk": lambda: e.infer_device(dx, n, sc)}
    ms = {k: [] for k in calls}
    for r in range(reps + 1):
        for k, fn in calls.items():
            t = event_ms(fn)
            if r:
                ms[k].append(t)
    for k in calls:
        m = float(np.median(ms[k]))
        res[k] = {"ms": m, "tuples_per_s": n / (m * 1e-3), "runs_ms": ms[k]}
        progress("%s %s: %.3g tuples/s" % (tag, k, res[k]["tuples_per_s"]))
    p1, p2 = pass_split(calls["approx"])
    res["pass_split_profiler_ms"] = {"pass1_leaf_walk": p1, "pass2_dt_approx_generic": p2,
                                     "pass2_share": p2 / (p1 + p2) if p1 + p2 else None}
    res["approx_over_score_time"] = res["approx"]["ms"] / res["score_walk"]["ms"]
    res["pass2_model_per_tuple"] = {"fp64_adds": Tu * (D + 1), "table_load_bytes": Tu * (D * 10 + 8),
                                    "accumulator_bytes": Tu * (D + 1) * 16 + (F + 1) * 20, "cell_bytes": 2 * Tu}
    # checks: efficiency on every tuple, words of a sample against approx_ref
    n_int = (1 << D) - 1
    leaf_abs = float(np.abs(W[:Tu, n_int:].view(np.float32).astype(np.float64)).max(axis=1).sum())
    e.infer_device_approx_contribs(dx, n, out)
    e.infer_device(dx, n, sc)
    p = out.double()
    bound = U * p.abs().sum(dim=1) + (Tu + 1) * U * leaf_abs + 1e-12 * leaf_abs
    eff_ok = bool(((p.sum(dim=1) - sc.double()).abs() <= bound).all().item())
    del p
    xs = L.synth_tuples(0, sample, F, seed=SEED, missing_ppm=MISSING_PPM)
    want = approx_contribs(W, FI, cov, xs, D, F, ntrees=Tu)[:, 0, :]
    words_ok = bool((out[:sample].cpu().numpy().view(np.uint32) == want.view(np.uint32)).all())
    res["efficiency_every_tuple"] = eff_ok
    res["words_equal_approx_ref_sample"] = words_ok
    e.close()
    if not (eff_ok and words_ok):
        raise SystemExit("%s: check failed (efficiency %s, words %s)" % (tag, eff_ok, words_ok))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sample", type=int, default=64)
    ap.add_argument("--tuples", type=int, default=2_000_000)
    ap.add_argument("--only", default="cfg2,cfg4_shard,cfg3")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power, max_sm, sm = card()
    line = {"what": "approximate contributions (dte_infer_device_approx_contribs) against the leaf and score walks on the "
                    "same handle", "card": name, "power_limit": power, "max_sm_clock": max_sm, "sm_clock_at_start": sm,
            "workloads": {tag: run(tag, a.reps, a.sample, a.tuples) for tag in a.only.split(",")}}
    line["sm_clock_at_end"] = card()[3]
    s = json.dumps(line)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
