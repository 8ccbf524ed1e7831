"""Leaf-index inference against the score walk on one H100: prints one JSON line.

Workloads: bench.py's ensembles, tuples and seeds (K = 8): cfg3 (1024 trees, D = 12, F = 256, 50 M tuples resident),
cfg2 (512 trees, D = 8, F = 128, 10 M) and the cfg4 shard (1024 trees, D = 10, F = 256, 20 M, ensemble seed 0xE5E).
Per workload, on one handle loaded with the leaf-id layout and the paths alternated:
  * device-resident walks: dte_infer_device over the resident tuples against dte_infer_device_leaves over the same
    tuples, median of --reps.  cfg3's 50 M tuples (51 GB) and their 102 GB of cells do not fit one 80 GB card together,
    so the leaf walk runs over the resident tuples in chunks of --chunk tuples into one reused output buffer; the time
    is that of all chunks;
  * host paths from pinned buffers on --host-tuples tuples: dte_infer_host against dte_infer_host_leaves.
Every run checks the cells of a 4096-tuple sample against the host leaf-cell walker (tests/leaf_oracle.py) and, on the
full output, the scores rebuilt from the cells (leaf values, tree8 / slot / cluster order, add.rn.ftz) against the
score walk's words.  The card name and power limit are printed with the numbers.  bench.py is not involved.
    python tools/bench_leaves.py [--reps 3] [--host-tuples 4000000] [--only cfg3,cfg2,cfg4_shard] [--out FILE] [--lib SO]"""
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
from leaf_oracle import leaf_cells  # noqa: E402

L = ddt.layout
SEED = 0x7091E5
MISSING_PPM = 10000
K = 8
WORKLOADS = {"cfg3": (1024, 12, 256, 50_000_000, None), "cfg2": (512, 8, 128, 10_000_000, None),
             "cfg4_shard": (1024, 10, 256, 20_000_000, 0xE5E)}
FLT_MIN = 1.1754943508222875e-38


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


def fadd(a, b):
    """add.rn.ftz.f32 on torch fp32 tensors: IEEE round-to-nearest, a subnormal result flushed to a signed zero (the
    leaf words are normal numbers, so no input is subnormal)."""
    r = a + b
    return torch.where(r.abs() < FLT_MIN, torch.zeros_like(r).copysign(r), r)


def rebuilt_scores(Wt, cells, T, S):
    """Scores from cells [m, T] (int16 on the device): leaf words, then the engine's tree8 / slot / cluster order."""
    m = cells.shape[0]
    v = torch.zeros((m, S * K * 8), dtype=torch.float32, device="cuda")
    v[:, :T] = Wt[torch.arange(T, device="cuda")[None, :], cells.long() & 0xFFFF]
    l = v.view(m, S, K, 8)
    r = fadd(fadd(fadd(l[..., 0], l[..., 1]), fadd(l[..., 2], l[..., 3])), fadd(fadd(l[..., 4], l[..., 5]), fadd(l[..., 6], l[..., 7])))
    acc = torch.zeros((m, K), dtype=torch.float32, device="cuda")
    for s in range(S):
        acc = fadd(r[:, s, :], acc)
    tot = torch.zeros(m, dtype=torch.float32, device="cuda")
    for j in range(K):
        tot = fadd(acc[:, j], tot)
    return tot


def run(tag, T, D, F, n, seed, reps, n_host, chunk):
    W, FI = L.synth_ensemble(T, D, F) if seed is None else L.synth_ensemble(T, D, F, seed=seed)
    wl, fl = L.pack_streams(W, FI, D)
    S = -(-T // (8 * K))
    e = ddt.Engine(0)
    e.configure(T, D, 4 * F, clusters=K, missing_value=L.MISSING_DEFAULT, n_tuples=n)
    e.load_ensemble(wl, fl, leaves=True)
    st = torch.cuda.current_stream().cuda_stream
    d_x = torch.empty((n, F), dtype=torch.int32, device="cuda")
    e.synth_tuples_device(d_x, 0, n, F, SEED, MISSING_PPM, L.MISSING_DEFAULT, stream=st)
    d_s = torch.empty(n, dtype=torch.float32, device="cuda")
    chunk = min(chunk, n)
    d_c = torch.empty((chunk, T), dtype=torch.int16, device="cuda")

    def score():
        e.infer_device(d_x, n, d_s, stream=st)

    def leaves(check=None):
        for a in range(0, n, chunk):
            m = min(chunk, n - a)
            e.infer_device_leaves(d_x[a:a + m], m, d_c[:m], stream=st)
            if check is not None:
                check(a, m)

    t_s, t_l = [], []
    for _ in range(reps):
        t_s.append(timed(score))
        t_l.append(timed(leaves))
    # checks: the full output against the rebuilt scores, a sample against the host walker
    Wt = torch.from_numpy(W.view(np.float32)).cuda()
    bad = [0]
    sub = 1 << 18

    def check(a, m):
        for b in range(0, m, sub):
            k = min(sub, m - b)
            got = rebuilt_scores(Wt, d_c[b:b + k], T, S).view(torch.int32)
            bad[0] += int((got != d_s[a + b:a + b + k].view(torch.int32)).sum())

    leaves(check)
    rng = np.random.default_rng(0x1EAF)
    idx = np.sort(rng.choice(n, 4096, replace=False))
    xs = np.stack([L.synth_tuples(int(i), 1, F, seed=SEED, missing_ppm=MISSING_PPM)[0] for i in idx])
    want = leaf_cells(W, FI, xs, D, L.MISSING_DEFAULT)
    got = np.empty_like(want)
    for a in range(0, n, chunk):                           # the sampled rows of every chunk
        m = min(chunk, n - a)
        sel = (idx >= a) & (idx < a + m)
        if sel.any():
            e.infer_device_leaves(d_x[a:a + m], m, d_c[:m], stream=st)
            torch.cuda.synchronize()
            got[sel] = d_c[torch.from_numpy(idx[sel] - a).cuda()].cpu().numpy().view(np.uint16)
    sample_ok = bool((got == want).all())
    name_s, name_l = e.kernel_name(), e.kernel_name_leaves()
    del d_x, d_s, d_c
    torch.cuda.empty_cache()

    # host paths from pinned buffers
    nh = min(n_host, n)
    h_x = torch.from_numpy(L.synth_tuples(0, nh, F, seed=SEED, missing_ppm=MISSING_PPM).view(np.int32)).pin_memory()
    h_s = torch.empty(nh, dtype=torch.float32).pin_memory()
    h_l = torch.empty(nh, dtype=torch.uint8).pin_memory()
    h_c = torch.empty((nh, T), dtype=torch.int16).pin_memory()
    th_s, th_l = [], []
    for _ in range(reps):
        th_s.append(timed(lambda: e.infer_host(h_x, out_scores=h_s.numpy(), out_labels=h_l.numpy())))
        th_l.append(timed(lambda: e.infer_host_leaves(h_x, out=h_c.numpy())))
    host_ok = bool((h_c.numpy().view(np.uint16)[idx[idx < nh]] == want[idx < nh]).all())
    e.close()
    ms_s, ms_l = float(np.median(t_s)), float(np.median(t_l))
    return {"workload": tag, "trees": T, "depth": D, "features": F, "tuples": n, "leaf_chunk_tuples": chunk,
            "score_walk_Mtps": n / ms_s / 1e3, "leaf_walk_Mtps": n / ms_l / 1e3, "leaf_over_score": ms_s / ms_l,
            "score_ms": t_s, "leaf_ms": t_l,
            "host_tuples": nh, "host_score_Mtps": nh / float(np.median(th_s)) / 1e3,
            "host_leaf_Mtps": nh / float(np.median(th_l)) / 1e3,
            "rebuilt_score_words_differing": bad[0], "oracle_sample_equal": sample_ok, "host_sample_equal": host_ok,
            "score_kernel": name_s, "leaf_kernel": name_l}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-tuples", type=int, default=4_000_000)
    ap.add_argument("--chunk", type=int, default=4_000_000)
    ap.add_argument("--only", default=",".join(WORKLOADS))
    ap.add_argument("--out", default=None)
    ap.add_argument("--lib", default=None, help="walk with this build of libdte.so instead of the in-tree one, e.g. the "
                    "store-ablation build of DESIGN.md §10")
    args = ap.parse_args()
    if args.lib:
        ddt.engine.lib_path = lambda: os.path.abspath(args.lib)
    name, power = card()
    res = {"card": name, "power_limit": power, "lib": args.lib or ddt.engine.lib_path(), "results": []}
    for tag in args.only.split(","):
        T, D, F, n, seed = WORKLOADS[tag]
        r = run(tag, T, D, F, n, seed, args.reps, args.host_tuples, args.chunk)
        res["results"].append(r)
        print(json.dumps(r), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
