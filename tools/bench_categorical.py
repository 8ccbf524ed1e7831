"""The categorical walk (DESIGN.md §16) against the fp32 walk on one H100: prints one JSON line.

Workloads: bench.py's ensembles (K = 8): cfg2 (512 trees, D = 8, F = 128), the cfg4 shard (1024 trees, D = 10, F = 256,
ensemble seed 0xE5E) and cfg3 (1024 trees, D = 12, F = 256).  Per workload, over --tuples device-resident tuples
(dte_synth_tuples_device, the seed bench.py uses):
  1. categorical: a quarter of the features categorical (every fourth), a quarter of the live nodes categorical on them
     (layout.synth_categorical), C_f categories per feature for each --categories value; the categorical columns of the
     tuples hold uniform codes 0 .. C_f - 1 (missing words stay missing).  dte_infer_device_categorical, median of --reps
     CUDA-event timings after one warm-up call;
  2. the same plain ensemble loaded with n_sets = 0: dte_infer_device_categorical against dte_infer_device on a plain load
     (the cost of the categorical-capable kernel on numeric trees);
  3. dte_infer_host_categorical from pinned host tuples (--host-tuples), wall time of one call after a warm-up;
  4. --sample tuples of the C_f = 100 ensemble checked word for word: each tree's leaf word is the oracle's score of that
     tree alone on its indicator expansion (tests/cat_ref.oracle_expanded), summed in the walk's order (cat_ref.sum_trees,
     held to the oracle by tests/test_cat_ref.py);
  5. the card name and power limit, read in the same run.
    python tools/bench_categorical.py [--tuples N] [--reps 5] [--categories 4,100,1000] [--only cfg2,cfg4_shard,cfg3]"""
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
from cat_ref import oracle_expanded, sum_trees  # noqa: E402

L = ddt.layout
SEED = 0x7091E5
MISSING_PPM = 10000
K = 8
WORKLOADS = {"cfg2": (512, 8, 128, None), "cfg4_shard": (1024, 10, 256, 0xE5E), "cfg3": (1024, 12, 256, None)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return [s.strip() for s in out.split(",")]
    except Exception:
        return [torch.cuda.get_device_name(0), "unknown", "unknown"]


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
    fn()
    return float(np.median([event_ms(fn) for _ in range(reps)]))


def sample_check(W, FI, x, D, S, off, words):
    """Score words of x by the oracle on each tree's expansion, summed in the walk's order (the first 8 S K trees)."""
    T = min(W.shape[0], 8 * S * K)
    leaves = np.zeros((x.shape[0], -(-T // 8) * 8), dtype=np.uint32)
    for t in range(T):
        leaves[:, t] = oracle_expanded(W[t:t + 1], FI[t:t + 1], x, D, 1, 1, L.MISSING_DEFAULT, off, words)
    return sum_trees(leaves, K, -(-T // 8))


def run(tag, args, cats):
    T, D, F, seed = WORKLOADS[tag]
    W, FI = L.synth_ensemble(T, D, F) if seed is None else L.synth_ensemble(T, D, F, seed=seed)
    wl, fl = L.pack_streams(W, FI, D)
    S = max(1, -(-T // (8 * K)))
    n = args.tuples
    e = ddt.Engine(0)
    e.configure(T, D, 4 * F, clusters=K)
    dx = torch.empty((n, F), dtype=torch.float32, device="cuda")
    e.synth_tuples_device(dx, 0, n, F, SEED, MISSING_PPM, L.MISSING_DEFAULT)
    sc = torch.empty(n, dtype=torch.float32, device="cuda")
    res = {"trees": T, "D": D, "F": F, "tuples": n}
    # 2. numeric trees: the fp32 walk, then the categorical walk on the same trees with no sets
    e.load_ensemble(wl, fl)
    res["fp32_kernel"] = e.kernel_name()
    res["fp32_ms"] = timed(lambda: e.infer_device(dx, n, sc), args.reps)
    plain = sc.clone()
    e.load_ensemble(wl, fl, categories=(None, None))
    res["no_sets_kernel"] = e.kernel_name_categorical()
    res["no_sets_ms"] = timed(lambda: e.infer_device_categorical(dx, n, sc), args.reps)
    res["no_sets_equal_words"] = bool(torch.equal(sc.view(torch.int32), plain.view(torch.int32)))
    res["no_sets_over_fp32"] = res["no_sets_ms"] / res["fp32_ms"]
    progress("%s: fp32 %.3f ms, categorical walk with no sets %.3f ms (%.2fx)" % (tag, res["fp32_ms"], res["no_sets_ms"],
                                                                                 res["no_sets_over_fp32"]))
    # 1. a quarter of the features categorical
    cat_f = np.arange(0, F, 4)
    res["categorical"] = {}
    for cf in cats:
        Wc, FIc, off, words = L.synth_categorical(W, FI, D, cat_f, cf, share=0.25, seed=0xCA7 + cf)
        t0 = time.perf_counter()
        e.load_ensemble(*L.pack_streams(Wc, FIc, D), categories=(off, words))
        load_s = time.perf_counter() - t0
        xc = dx.clone()
        g = torch.Generator(device="cuda").manual_seed(cf)
        for f in cat_f:
            col = xc[:, int(f)]
            codes = torch.randint(0, cf, (n,), device="cuda", generator=g).to(torch.float32)
            xc[:, int(f)] = torch.where(col.view(torch.int32) == np.int32(np.uint32(L.MISSING_DEFAULT).view(np.int32)), col, codes)
        ms = timed(lambda: e.infer_device_categorical(xc, n, sc), args.reps)
        r = {"kernel": e.kernel_name_categorical(), "n_sets": int(off.size - 1), "set_words": int(words.size),
             "load_s": load_s, "ms": ms, "tuples_per_s": n / (ms * 1e-3), "over_fp32": ms / res["fp32_ms"]}
        if cf == 100:
            # 3. pinned host tuples
            nh = min(n, args.host_tuples)
            hx = e.host_alloc((nh, F), np.float32)
            hx[:] = xc[:nh].cpu().numpy()
            hs = e.host_alloc((nh,), np.float32)
            e.infer_host_categorical(hx, want_labels=False, out_scores=hs)
            t0 = time.perf_counter()
            e.infer_host_categorical(hx, want_labels=False, out_scores=hs)
            r["host_pinned_tuples_per_s"] = nh / (time.perf_counter() - t0)
            # 4. sampled comparison against the oracle on the expansion
            idx = np.random.default_rng(7).choice(n, size=args.sample, replace=False)
            xs = xc[torch.from_numpy(idx).cuda()].cpu().numpy().view(np.uint32)
            want = sample_check(Wc, FIc, xs, D, S, off, words)
            got = sc[torch.from_numpy(idx).cuda()].cpu().numpy().view(np.uint32)
            e.infer_device_categorical(xc, n, sc)
            got = sc[torch.from_numpy(idx).cuda()].cpu().numpy().view(np.uint32)
            r["sample_checked"] = int(args.sample)
            r["sample_equal"] = int((got == want).sum())
            r["host_sample_equal"] = int((hs.view(np.uint32)[idx[idx < nh]] == want[idx < nh]).sum())
            r["host_sample_checked"] = int((idx < nh).sum())
            e.host_free(hx)
            e.host_free(hs)
        progress("%s C_f=%d: %s %.4g tuples/s (%.2fx the fp32 walk)%s" % (
            tag, cf, r["kernel"], r["tuples_per_s"], r["over_fp32"],
            " sample %d/%d equal" % (r["sample_equal"], r["sample_checked"]) if "sample_equal" in r else ""))
        res["categorical"][str(cf)] = r
    e.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tuples", type=int, default=1 << 21)
    ap.add_argument("--host-tuples", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sample", type=int, default=128)
    ap.add_argument("--categories", default="4,100,1000")
    ap.add_argument("--only", default="cfg2,cfg4_shard,cfg3")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    cats = [int(c) for c in args.categories.split(",")]
    if 100 not in cats:
        cats.append(100)
    name, power, sm_max = card()
    line = {"bench": "categorical", "card": name, "power_limit": power, "sm_clock_max": sm_max, "workloads": {}}
    for tag in args.only.split(","):
        line["workloads"][tag] = run(tag, args, cats)
    s = json.dumps(line)
    print(s)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(s + "\n")


if __name__ == "__main__":
    main()
