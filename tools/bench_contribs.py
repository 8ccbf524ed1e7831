"""TreeSHAP feature contributions against the score walk on one H100: prints one JSON line.

Workloads: bench.py's ensembles and tuple seeds (K = 8) with layout.synth_covers: cfg2 (512 trees, D = 8, F = 128), the
cfg4 shard (1024 trees, D = 10, F = 256, ensemble seed 0xE5E) and cfg3 (1024 trees, D = 12, F = 256).  Per workload, on
one handle loaded with the contribution layout, over the same device-resident synthetic tuples (two waves of the tile
kernel's CTAs, one at cfg3; --tuples overrides): dte_infer_device_contribs with the tile kernel (DTE_KERNEL_TILE) and
with the generic kernel (DTE_KERNEL_GENERIC), median of --reps each after one warm-up run; the kernel AUTO takes is
reported too.  The score walk (dte_infer_device) on the same handle is timed on --score-tuples tuples of the same set, so
that its time is the walk's and not the launch's.

Checks on every run: efficiency on every tuple (sum_f phi + bias against the same handle's score word, within
U sum|phi| + (T + 1) U sum_t max|leaf_t|, U = 2^-24), and word equality of --sample tuples with
tests/shap_ref.path_treeshap, for both kernels.

fp64 operations per tuple are a model figure counted from the path layout, as the kernels issue them (both sides of the
per-lane o branch, since a warp executes them predicated): per path of m merged elements 4 m (m + 1) / 2 for the extend,
m (7 m + 5) for the unwound sums, contributions and accumulations, and 1 for the bias.  The achieved rate is given as a
fraction of the H100 SXM data-sheet fp64 (non-tensor) figure, 34 TFLOP/s.
    python tools/bench_contribs.py [--reps 3] [--sample 4] [--only cfg2,cfg4_shard,cfg3] [--out FILE]"""
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
from ddt_b200 import engine as E  # noqa: E402
from shap_ref import path_treeshap, tree_paths  # noqa: E402

L = ddt.layout
SEED = 0x7091E5
MISSING_PPM = 10000
K = 8
H100_SXM_FP64 = 34e12          # data-sheet fp64 (non-tensor) FLOP/s of the H100 SXM
U = 2.0 ** -24
# (trees, D, F, ensemble seed, waves of tile CTAs timed)
WORKLOADS = {"cfg2": (512, 8, 128, None, 2), "cfg4_shard": (1024, 10, 256, 0xE5E, 2), "cfg3": (1024, 12, 256, None, 1)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def progress(*a):
    print(*a, file=sys.stderr, flush=True)


def timed(fn, reps):
    ms = []
    for _ in range(reps + 1):                        # the first run is a warm-up
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms[1:]))


def ops_per_tuple(W, FI, cov, D):
    total = 0
    for t in range(W.shape[0]):
        m = tree_paths(W[t], FI[t], cov[t], D)["m"].astype(np.int64)
        total += int((2 * m * (m + 1) + m * (7 * m + 5) + 1).sum())
    return total


def run(tag, reps, sample, n_override, n_score):
    T, D, F, seed, waves = WORKLOADS[tag]
    W, FI = L.synth_ensemble(T, D, F) if seed is None else L.synth_ensemble(T, D, F, seed=seed)
    cov = L.synth_covers(FI, D)
    wl, fl = L.pack_streams(W, FI, D)
    e = ddt.Engine(0)
    e.configure(T, D, 4 * F, clusters=K)
    e.load_ensemble(wl, fl, covers=cov)
    info = e.info()
    kernel_auto = e.kernel_name_contribs()
    e.set_kernel_variant(E.DTE_KERNEL_TILE)
    name_tile = e.kernel_name_contribs()
    groups = int(name_tile.split("warps=")[1].split()[0]) if "warps=" in name_tile else 1
    n = n_override or waves * info["sm_count"] * 32 * groups
    dx = torch.empty((n, F), dtype=torch.float32, device="cuda")
    e.synth_tuples_device(dx, 0, n, F, SEED, MISSING_PPM, L.MISSING_DEFAULT)
    torch.cuda.synchronize()
    out = torch.empty((n, F + 1), dtype=torch.float32, device="cuda")
    sc = torch.empty(n, dtype=torch.float32, device="cuda")
    res = {"trees": T, "D": D, "F": F, "tuples": n, "kernel_tile": name_tile, "kernel_auto": kernel_auto,
           "contrib_layout_bytes": int(info["ensemble_bytes"])}
    n_int = (1 << D) - 1
    leaf_abs = float(np.abs(W[:, n_int:].view(np.float32).astype(np.float64)).max(axis=1).sum())
    xs = L.synth_tuples(0, sample, F, seed=SEED, missing_ppm=MISSING_PPM)
    want = path_treeshap(W, FI, cov, xs, D, F)[:, 0, :]
    progress("%s: %d tuples, %s, reference sample done" % (tag, n, name_tile))
    e.infer_device(dx, n, sc)
    score = sc.double()
    for kind, variant in (("tile", E.DTE_KERNEL_TILE), ("generic", E.DTE_KERNEL_GENERIC)):
        e.set_kernel_variant(variant)
        ms = timed(lambda: e.infer_device_contribs(dx, n, out), reps)
        p = out.double()
        bound = U * p.abs().sum(dim=1) + (T + 1) * U * leaf_abs
        eff_ok = bool(((p.sum(dim=1) - score).abs() <= bound).all().item())
        words_ok = bool((out[:sample].cpu().numpy().view(np.uint32) == want.view(np.uint32)).all())
        res[kind] = {"tuples_per_s": n / (ms * 1e-3), "ms": ms, "efficiency_every_tuple": eff_ok,
                     "words_equal_path_treeshap_sample": words_ok}
        progress("%s %s: %.1f tuples/s" % (tag, kind, res[kind]["tuples_per_s"]))
        if not (eff_ok and words_ok):
            raise SystemExit("%s %s: check failed (efficiency %s, words %s)" % (tag, kind, eff_ok, words_ok))
    res["kernel_generic"] = e.kernel_name_contribs()
    e.set_kernel_variant(E.DTE_KERNEL_AUTO)
    del dx, out, sc, p
    dxs = torch.empty((n_score, F), dtype=torch.float32, device="cuda")
    e.synth_tuples_device(dxs, 0, n_score, F, SEED, MISSING_PPM, L.MISSING_DEFAULT)
    scs = torch.empty(n_score, dtype=torch.float32, device="cuda")
    ms_score = timed(lambda: e.infer_device(dxs, n_score, scs), reps)
    res["score_walk"] = {"tuples": n_score, "tuples_per_s": n_score / (ms_score * 1e-3), "ms": ms_score}
    best = max(res["tile"]["tuples_per_s"], res["generic"]["tuples_per_s"])
    res["score_over_contrib_rate"] = res["score_walk"]["tuples_per_s"] / best
    ops = ops_per_tuple(W, FI, cov, D)
    res["fp64_ops_per_tuple_model"] = ops
    res["fp64_fraction_of_datasheet_model"] = {k: ops * res[k]["tuples_per_s"] / H100_SXM_FP64 for k in ("tile", "generic")}
    e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sample", type=int, default=4)
    ap.add_argument("--tuples", type=int, default=0)
    ap.add_argument("--score-tuples", type=int, default=4_000_000)
    ap.add_argument("--only", default="cfg2,cfg4_shard,cfg3")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    line = {"what": "TreeSHAP contributions (dte_infer_device_contribs) against the score walk on the same handle",
            "card": name, "power_limit": power, "fp64_reference": "H100 SXM data sheet, fp64 non-tensor, 34 TFLOP/s (model figure)",
            "workloads": {tag: run(tag, a.reps, a.sample, a.tuples, a.score_tuples) for tag in a.only.split(",")}}
    s = json.dumps(line)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
