"""Interventional SHAP values against the score walk and TreeSHAP on one H100: prints one JSON line.

Workloads: bench.py's ensembles and tuple seeds (K = 8): cfg2 (512 trees, D = 8, F = 128), the cfg4 shard (1024 trees,
D = 10, F = 256, ensemble seed 0xE5E) and cfg3 (1024 trees, D = 12, F = 256), each with N = 100 background rows, and
cfg2 with N = 1000 ("cfg2_N1000").  The background rows are layout.synth_tuples rows of another seed (BG_SEED).

Per workload, over the same device-resident synthetic tuples: --warps-per-sm (8 by default) warps of 32 tuples for
every SM of the card, so both attribution kernels (128-thread blocks, one lane per tuple) spread over every SM, two
blocks each at the default (33,792 tuples on 132 SMs); --tuples overrides.
  - the load: wall time of load_ensemble(..., background=bg) (path layout built on the host, then uploaded);
  - dte_infer_device_interventional, dte_infer_device (the score walk) and, on a second handle loaded with covers
    (layout.synth_covers), dte_infer_device_contribs (TreeSHAP, §12, the kernel AUTO takes), each timed with CUDA events
    around one call, --reps times (median and every run reported).  The attribution calls take seconds, so they get no
    warm-up call of their own; the first launch of a kernel module costs milliseconds, which the spread shows.

Operation-count model kept here: (path, background-row) pairs per tuple = sum_t paths_t * N (complete trees: 2^D paths
per tree, the trees the run adds), and per pair the kernel does one mask merge and up to M 32-bit additions, plus one
D-step walk per path and block of 32 rows for the row masks.

Checks on every run: efficiency on every timed tuple (sum_f phi + bias against the same handle's score word, within
U sum|phi| + (T + 1) U sum_t max|leaf_t| + 1e-12 sum_t max|leaf_t|, U = 2^-24), and --sample tuples word for word against
tests/interv_ref.interventional on a run that adds the first 8 trees (K = S = 1 written to register 205 of the same
handle: a run's K and S are free to change, and the whole restatement of a 1024-tree ensemble takes minutes on a CPU).
    python tools/bench_interventional.py [--reps 2] [--warps-per-sm 8] [--tuples N] [--sample 4]
                                         [--only cfg2,cfg2_N1000,cfg4_shard,cfg3] [--out F]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import ddt_b200 as ddt  # noqa: E402
from helpers import geometry_regs  # noqa: E402
from interv_ref import interventional  # noqa: E402

L = ddt.layout
SEED = 0x7091E5
BG_SEED = 0xB6E5
MISSING_PPM = 10000
K = 8
U = 2.0 ** -24
WORKLOADS = {"cfg2": (512, 8, 128, None, 100), "cfg2_N1000": (512, 8, 128, None, 1000),
             "cfg4_shard": (1024, 10, 256, 0xE5E, 100), "cfg3": (1024, 12, 256, None, 100)}


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


def timed(fn, reps):
    runs = [event_ms(fn) for _ in range(reps)]
    return float(np.median(runs)), runs


def run(tag, reps, sample, n):
    T, D, F, seed, N = WORKLOADS[tag]
    W, FI = L.synth_ensemble(T, D, F) if seed is None else L.synth_ensemble(T, D, F, seed=seed)
    wl, fl = L.pack_streams(W, FI, D)
    bg = L.synth_tuples(0, N, F, seed=BG_SEED, missing_ppm=MISSING_PPM)
    S = max(1, -(-T // (8 * K)))
    Tu = min(T, 8 * K * S)
    e = ddt.Engine(0)
    e.configure(T, D, 4 * F, clusters=K)
    t0 = time.perf_counter()
    e.load_ensemble(wl, fl, background=bg)
    load_s = time.perf_counter() - t0
    dx = torch.empty((n, F), dtype=torch.float32, device="cuda")
    e.synth_tuples_device(dx, 0, n, F, SEED, MISSING_PPM, L.MISSING_DEFAULT)
    out = torch.empty((n, F + 1), dtype=torch.float32, device="cuda")
    sc = torch.empty(n, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    pairs = Tu * (1 << D) * N
    res = {"trees": T, "D": D, "F": F, "background_rows": N, "tuples": n, "kernel": e.kernel_name_interventional(),
           "layout_load_s": load_s, "ensemble_bytes": int(e.info()["ensemble_bytes"]),
           "model_path_row_pairs_per_tuple": pairs}
    progress("%s: %d tuples, %s, load %.2f s, %.3g pairs per tuple" % (tag, n, res["kernel"], load_s, pairs))
    event_ms(lambda: e.infer_device(dx, n, sc))                     # warm-up of the score walk
    res["score_walk_ms"] = event_ms(lambda: e.infer_device(dx, n, sc))
    res["interventional_ms"], res["interventional_runs_ms"] = timed(lambda: e.infer_device_interventional(dx, n, out), reps)
    res["interventional_tuples_per_s"] = n / (res["interventional_ms"] * 1e-3)
    res["model_path_row_pairs_per_s"] = pairs * n / (res["interventional_ms"] * 1e-3)
    progress("%s interventional: %.4g tuples/s" % (tag, res["interventional_tuples_per_s"]))
    # efficiency on every timed tuple
    leaf_abs = float(np.abs(W[:Tu, (1 << D) - 1:].view(np.float32).astype(np.float64)).max(axis=1).sum())
    p = out.double()
    bound = U * p.abs().sum(dim=1) + (Tu + 1) * U * leaf_abs + 1e-12 * leaf_abs
    eff_ok = bool(((p.sum(dim=1) - sc.double()).abs() <= bound).all().item())
    del p
    # a sample word for word, on a run adding the first 8 trees
    for a, v in sorted(geometry_regs(T, D, F, 1, 1, L.MISSING_DEFAULT).items()):
        e.softreg_write(a, v)
    xs = L.synth_tuples(0, sample, F, seed=SEED, missing_ppm=MISSING_PPM)
    got = e.infer_host_interventional(xs)
    want = interventional(W, FI, xs, bg, D, F, ntrees=8)[:, 0, :]
    words_ok = bool((got.view(np.uint32) == want.view(np.uint32)).all())
    e.close()
    if tag != "cfg2_N1000":                                          # TreeSHAP does not depend on N
        c = ddt.Engine(0)
        c.configure(T, D, 4 * F, clusters=K)
        c.load_ensemble(wl, fl, covers=L.synth_covers(FI, D))
        res["treeshap_kernel"] = c.kernel_name_contribs()
        res["treeshap_ms"], res["treeshap_runs_ms"] = timed(lambda: c.infer_device_contribs(dx, n, out), reps)
        res["treeshap_tuples_per_s"] = n / (res["treeshap_ms"] * 1e-3)
        res["interventional_over_treeshap_time"] = res["interventional_ms"] / res["treeshap_ms"]
        c.close()
        progress("%s treeshap: %.4g tuples/s" % (tag, res["treeshap_tuples_per_s"]))
    res["interventional_over_score_time"] = res["interventional_ms"] / res["score_walk_ms"]
    res["efficiency_every_tuple"] = eff_ok
    res["words_equal_interv_ref_sample_8_trees"] = words_ok
    if not (eff_ok and words_ok):
        raise SystemExit("%s: check failed (efficiency %s, words %s)" % (tag, eff_ok, words_ok))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--warps-per-sm", type=int, default=8)
    ap.add_argument("--sample", type=int, default=4)
    ap.add_argument("--tuples", type=int, default=0)
    ap.add_argument("--only", default="cfg2,cfg2_N1000,cfg4_shard,cfg3")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power, max_sm, sm = card()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = a.tuples or sms * 32 * a.warps_per_sm
    line = {"what": "interventional SHAP values (dte_infer_device_interventional) against the score walk and TreeSHAP",
            "card": name, "power_limit": power, "max_sm_clock": max_sm, "sm_clock_at_start": sm, "sm_count": sms,
            "blocks_per_sm": n / (128 * sms), "workloads": {tag: run(tag, a.reps, a.sample, n) for tag in a.only.split(",")}}
    line["sm_clock_at_end"] = card()[3]
    s = json.dumps(line)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
