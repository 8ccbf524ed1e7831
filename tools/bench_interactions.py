"""SHAP interaction values against TreeSHAP contributions on one H100: prints one JSON line.

Workloads: bench.py's ensembles and tuple seeds (K = 8) with layout.synth_covers: cfg2 (512 trees, D = 8, F = 128), the
cfg4 shard (1024 trees, D = 10, F = 256, ensemble seed 0xE5E) and cfg3 (1024 trees, D = 12, F = 256) with few tuples.  Per
workload, on one handle loaded with the contribution layout, over the same device-resident synthetic tuples:
dte_infer_device_interactions and dte_infer_device_contribs (AUTO kernel), median of --reps each after one warm-up run.

Checks on every run: every row of every tuple sums (fp64 over its fp32 words) to the contribution word within
2 U (sum_k |inter[a][k]| + |phi_a|) + 1e-12 sum_t max|leaf_t|, U = 2^-24, [F][F] equals the bias word bit for bit, and
on the workloads of --sample-on the first --sample tuples equal tests/shap_inter_ref.path_interactions word for word
(the numpy restatement takes minutes at cfg3's 4 M paths, so cfg3 is not sampled by default).

fp64 operations per tuple are a model figure counted from the path layout, as the kernels issue them (both sides of the
per-lane o branch): the contribution count of tools/bench_contribs.py per path of m merged elements, plus for each of its
m elements the extension over the other m - 1 (2 m (m - 1)), their m - 1 unwound sums and accumulations
((m - 1) (7 m - 2)) and 2 for v'.  It leaves out the re-extension of a path in every further pass that reaches it.
The achieved rate is given as a fraction of the H100 SXM data-sheet fp64 (non-tensor) figure, 34 TFLOP/s.
Only cfg2 runs by default: at these tuple counts (a few warps per SM) the cfg4 shard and cfg3 take minutes per call.
    python tools/bench_interactions.py [--reps 3] [--sample 2] [--only cfg2,cfg4_shard,cfg3] [--out FILE]"""
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
from shap_inter_ref import path_interactions  # noqa: E402
from shap_ref import tree_paths  # noqa: E402

L = ddt.layout
SEED = 0x7091E5
MISSING_PPM = 10000
K = 8
H100_SXM_FP64 = 34e12          # data-sheet fp64 (non-tensor) FLOP/s of the H100 SXM
U = 2.0 ** -24
# (trees, D, F, ensemble seed, tuples per SM timed)
WORKLOADS = {"cfg2": (512, 8, 128, None, 64), "cfg4_shard": (1024, 10, 256, 0xE5E, 4), "cfg3": (1024, 12, 256, None, 1)}


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
    contrib = inter = 0
    for t in range(W.shape[0]):
        m = tree_paths(W[t], FI[t], cov[t], D)["m"].astype(np.int64)
        contrib += int((2 * m * (m + 1) + m * (7 * m + 5) + 1).sum())
        inter += int((m * (2 * m * (m - 1) + (m - 1) * (7 * m - 2) + 2)).sum())
    return contrib, contrib + inter


def run(tag, reps, sample):
    T, D, F, seed, per_sm = WORKLOADS[tag]
    W, FI = L.synth_ensemble(T, D, F) if seed is None else L.synth_ensemble(T, D, F, seed=seed)
    cov = L.synth_covers(FI, D)
    wl, fl = L.pack_streams(W, FI, D)
    e = ddt.Engine(0)
    e.configure(T, D, 4 * F, clusters=K)
    e.load_ensemble(wl, fl, covers=cov)
    info = e.info()
    n = per_sm * info["sm_count"]
    dx = torch.empty((n, F), dtype=torch.float32, device="cuda")
    e.synth_tuples_device(dx, 0, n, F, SEED, MISSING_PPM, L.MISSING_DEFAULT)
    inter = torch.empty((n, F + 1, F + 1), dtype=torch.float32, device="cuda")
    phi = torch.empty((n, F + 1), dtype=torch.float32, device="cuda")
    res = {"trees": T, "D": D, "F": F, "tuples": n, "kernel": e.kernel_name_interactions(),
           "kernel_contribs": e.kernel_name_contribs(), "contrib_layout_bytes": int(info["ensemble_bytes"])}
    progress("%s: %d tuples, %s" % (tag, n, res["kernel"]))
    ms_c = timed(lambda: e.infer_device_contribs(dx, n, phi), reps)
    launches = e.info()["kernel_launches"]
    ms_i = timed(lambda: e.infer_device_interactions(dx, n, inter), reps)
    res["launches_per_call"] = (e.info()["kernel_launches"] - launches) // (reps + 1)
    out_bytes = n * (F + 1) * (F + 1) * 4
    res["interactions"] = {"tuples_per_s": n / (ms_i * 1e-3), "ms": ms_i, "output_GB_per_s": out_bytes / (ms_i * 1e-3) / 1e9}
    res["contribs"] = {"tuples_per_s": n / (ms_c * 1e-3), "ms": ms_c}
    res["contrib_over_inter_rate"] = res["contribs"]["tuples_per_s"] / res["interactions"]["tuples_per_s"]
    progress("%s: interactions %.1f tuples/s, contributions %.1f tuples/s" % (tag, res["interactions"]["tuples_per_s"],
                                                                               res["contribs"]["tuples_per_s"]))
    n_int = (1 << D) - 1
    leaf_abs = float(np.abs(W[:, n_int:].view(np.float32).astype(np.float64)).max(axis=1).sum())
    ok_rows, ok_bias = True, True
    for a in range(0, n, 256):                      # on the device, a slice of tuples at a time
        p = inter[a:a + 256].double()
        c = phi[a:a + 256].double()
        rows = p[:, :F, :].sum(dim=2)
        bound = 2 * U * (p[:, :F, :].abs().sum(dim=2) + c[:, :F].abs()) + 1e-12 * leaf_abs
        ok_rows &= bool(((rows - c[:, :F]).abs() <= bound).all().item())
        ok_bias &= bool(torch.equal(inter[a:a + 256, F, F].view(torch.int32), phi[a:a + 256, F].view(torch.int32)))
    res["row_sums_match_contribs"] = ok_rows
    res["bias_word_equal"] = ok_bias
    if sample:
        xs = L.synth_tuples(0, sample, F, seed=SEED, missing_ppm=MISSING_PPM)
        want = path_interactions(W, FI, cov, xs, D, F)[:, 0]
        res["words_equal_path_interactions_sample"] = bool(
            (inter[:sample].cpu().numpy().view(np.uint32) == want.view(np.uint32)).all())
    ops_c, ops_i = ops_per_tuple(W, FI, cov, D)
    res["fp64_ops_per_tuple_model"] = {"contribs": ops_c, "interactions": ops_i}
    res["fp64_fraction_of_datasheet_model"] = {"contribs": ops_c * res["contribs"]["tuples_per_s"] / H100_SXM_FP64,
                                               "interactions": ops_i * res["interactions"]["tuples_per_s"] / H100_SXM_FP64}
    e.close()
    del dx, inter, phi
    torch.cuda.empty_cache()
    if not (ok_rows and ok_bias and res.get("words_equal_path_interactions_sample", True)):
        raise SystemExit("%s: check failed: %s" % (tag, json.dumps(res)))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sample", type=int, default=2)
    ap.add_argument("--sample-on", default="cfg2")
    ap.add_argument("--only", default="cfg2")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    sampled = set(a.sample_on.split(","))
    line = {"what": "SHAP interaction values (dte_infer_device_interactions) against contributions on the same handle",
            "card": name, "power_limit": power, "fp64_reference": "H100 SXM data sheet, fp64 non-tensor, 34 TFLOP/s (model figure)",
            "workloads": {tag: run(tag, a.reps, a.sample if tag in sampled else 0) for tag in a.only.split(",")}}
    s = json.dumps(line)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
