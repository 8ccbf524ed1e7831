"""The staged walk with split tree tops (dt_walk_tile_split, DTE_TUNE tops=6): 6-byte records in two runs instead of
8-byte records.  The compare is unchanged, so every score word and label must equal those of the 8-byte staged plan of
the same ensemble and tuples, and the oracle's."""
import numpy as np
import pytest

import ddt_b200 as ddt
from edge_operands import MISSING_ROTATION, edge_ensemble, edge_tuples, with_early_leaves
from helpers import make_engine, oracle_cfg, torch_cuda, L  # noqa: F401 (torch_cuda: a fixture)
from oracle import oracle as O

pytestmark = pytest.mark.gpu


def run(monkeypatch, tune, W, FI, D, F, K, S, missing, x=None, n_of=None):
    """Scores, labels and kernel name of a handle created under DTE_TUNE=tune; x = n_of(tuples per CTA, SMs) tuples
    when x is None is built by the caller from the returned n."""
    monkeypatch.setenv("DTE_TUNE", tune)
    e = make_engine(W.shape[0], D, F, K, S, missing)
    try:
        e.load_ensemble(*L.pack_streams(W, FI, D))
        info = e.info()
        if x is None:
            x = n_of(int(info["tuples_per_cta"]), int(info["sm_count"]))
        sc, lb = e.infer_host(x)
        return np.asarray(sc).view(np.uint32).copy(), np.asarray(lb).copy(), e.kernel_name(), x
    finally:
        e.close()


def check(monkeypatch, split_tune, byte8_tune, W, FI, D, F, K, S, missing, n_of, phased=None):
    s6, l6, name6, x = run(monkeypatch, split_tune, W, FI, D, F, K, S, missing, n_of=n_of)
    assert name6.endswith(" tops=6"), name6
    if phased is not None:
        assert (" phased=1 " in name6) == phased, name6
    s8, l8, name8, _ = run(monkeypatch, byte8_tune, W, FI, D, F, K, S, missing, x=x)
    assert "tops=6" not in name8, name8
    bad = np.flatnonzero(s6 != s8)
    assert bad.size == 0, "%s vs %s: %d words differ, first tuple %d" % (name6, name8, bad.size, bad[0])
    assert (l6 == l8).all(), name6
    idx = np.unique(np.linspace(0, x.shape[0] - 1, 512).astype(np.int64))
    want = O.scores(oracle_cfg(D, K, S, missing, F, W.shape[0]), *L.pack_streams(W, FI, D), x[idx], threads=O.max_threads())
    assert (s6[idx] == want).all(), "%s: %d / %d oracle words differ" % (name6, (s6[idx] != want).sum(), idx.size)
    return name6


def wave_edge(delta):
    return lambda per_cta, sms: per_cta * sms + delta


@pytest.mark.parametrize("D,F,early,delta", [
    (5, 64, False, 0), (8, 600, True, -1), (12, 256, True, 1), (12, 1024, False, 0), (14, 96, True, 33), (15, 32, False, -1),
], ids=["D5", "D8-wide-early", "D12-early", "D12-wide", "D14-early", "D15"])
def test_split_tops_against_the_8_byte_staged_plan(torch_cuda, monkeypatch, D, F, early, delta):
    """Unphased plans, compact (F <= 512) and wide records, early leaves inside the staged levels, n at wave edges.
    SP = 8 plans where a stage fits; from D = 14 only the SP = 4 families stage (D = 15: only with split tops, so the
    8-byte pin falls back to the non-staged tile walk, another independent layout)."""
    T, K, S = 32, 2, 2
    W, FI = L.synth_ensemble(T, D, F, seed=300 + D)
    if early:
        rng = np.random.default_rng(D)
        for t in range(T):
            for _ in range(3):
                lvl = int(rng.integers(0, D - 2))
                FI[t, (1 << lvl) - 1 + int(rng.integers(0, 1 << lvl))] |= 1 << 14
    base = "ilp=2,pair=4,stages=2,phased=0" if D <= 12 else "ilp=2,pair=2,stages=1,phased=0"

    def tuples(per_cta, sms):
        return L.synth_tuples(0, max(1, wave_edge(delta)(per_cta, sms)), F, seed=301 + D, missing_ppm=20000).view(np.uint32)

    check(monkeypatch, base + ",tops=6", base, W, FI, D, F, K, S, L.MISSING_DEFAULT, tuples, phased=False)


@pytest.mark.parametrize("D,tune,phased", [
    (7, "ilp=4,pair=2,stages=1,phased=1", True),          # Dtop = 5: the smallest phased level, Lw = 2
    (6, "ilp=4,pair=2,stages=1,phased=1", False),         # Lw = 1: the meta part A is no 16-byte unit, so unphased
    (12, "ilp=2,pair=4,stages=1,phased=1,warps=16", True),
    (12, "ilp=2,pair=4,stages=1,phased=3", True),         # part A ends two levels earlier
    (13, "ilp=2,pair=2,stages=2,phased=1", True),
], ids=["D7-Lw2", "D6-Lw1-off", "D12", "D12-phased3", "D13-2stages"])
def test_phased_split_tops(torch_cuda, monkeypatch, D, tune, phased):
    """The phased refill copies part A and part B of each tree as one piece of the threshold run and one of the meta
    run; the 8-byte reference is the same pin without tops=6."""
    T, K, S, F = 48, 2, 3, 128
    W, FI = L.synth_ensemble(T, D, F, seed=400 + D)

    def tuples(per_cta, sms):
        return L.synth_tuples(0, 2 * per_cta * sms + 7, F, seed=401 + D, missing_ppm=20000).view(np.uint32)

    check(monkeypatch, tune + ",tops=6", tune, W, FI, D, F, K, S, L.MISSING_DEFAULT, tuples, phased=phased)


@pytest.mark.parametrize("missing", MISSING_ROTATION)
def test_split_tops_on_edge_operands(torch_cuda, monkeypatch, missing):
    """Ties, sign-boundary words and the missing pattern at every level (tests/edge_operands.py), with early leaves."""
    T, D, F, K, S = 24, 9, 48, 1, 3
    W, FI, pools = edge_ensemble(T, D, F, seed=500, missing=missing)
    W, FI = with_early_leaves(W, FI, D, seed=501, root_trees=(2,))

    def tuples(per_cta, sms):
        return edge_tuples(per_cta * sms + 5, F, pools, seed=502, missing=missing)

    check(monkeypatch, "ilp=2,pair=4,stages=2,phased=0,tops=6", "ilp=2,pair=4,stages=2,phased=0", W, FI, D, F, K, S, missing,
          tuples)


def test_cfg3_large_workload_handle_runs_a_measured_plan_word_for_word(torch_cuda, monkeypatch):
    """cfg3 with the 50 M workload hint: the handle times the 8-byte and split-tops candidates at load and runs the
    fastest; 1 M tuples equal the static plan's words.  The stderr plan line and kernel_name() name the plan, with
    tops=6 when split tops run."""
    torch = torch_cuda
    monkeypatch.delenv("DTE_TUNE", raising=False)
    T, D, F, K = 1024, 12, 256, 8
    N = 1 << 20
    W, FI = L.synth_ensemble(T, D, F)
    wl, fl = L.pack_streams(W, FI, D)
    with ddt.Engine(0) as big, ddt.Engine(0) as small:
        big.configure(T, D, 4 * F, clusters=K, missing_value=L.MISSING_DEFAULT, n_tuples=50_000_000)
        big.load_ensemble(wl, fl)
        small.configure(T, D, 4 * F, clusters=K, missing_value=L.MISSING_DEFAULT, n_tuples=N)
        small.load_ensemble(wl, fl)
        name = big.kernel_name()
        print("\n[split-tops] measured plan: %s (%s)" % (name, big.info()["plan_source"]))
        assert "tops=6" not in small.kernel_name() and small.info()["plan_source"] == "static"
        d_x = torch.empty((N, F), dtype=torch.int32, device="cuda")
        small.synth_tuples_device(d_x, 0, N, F, 0x7091E5, 10000, L.MISSING_DEFAULT)
        s_big, s_small = (torch.empty(N, dtype=torch.float32, device="cuda") for _ in range(2))
        big.infer_device(d_x, N, s_big)
        small.infer_device(d_x, N, s_small)
        torch.cuda.synchronize()
        assert torch.equal(s_big.view(torch.int32), s_small.view(torch.int32)), name
