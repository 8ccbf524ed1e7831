"""Every walk kernel the planner can reach, and the edges of the supported domain, bit for bit against the oracle.

tests/golden/plan_table.txt.xz records the planner's choice for every DTE_TUNE pin, depth, feature count, class count
and requested variant (tests/test_plan_table.py keeps it equal to the planner).  The instantiation matrix below is
derived from it: the rows are grouped by (kernel template, C) and two rows of each group are run on the card with the
pin, geometry and variant of the row, so every reachable instantiation is launched and a kernel_name() that differs
from the table shows that the live planner (SM count, opt-in shared memory) disagrees with the recorded one.

The edge tests then drive single kernels to the depths, feature counts, record formats, tuple and tree counts, class
layouts, ring-fill knobs, pointer alignments and 64-bit offsets where a tile kernel could go wrong without the
headline geometry noticing.  Bar everywhere: every score word and every label equals the oracle's."""
import os
import re

import numpy as np
import pytest

from ddt_b200 import engine as E
from edge_operands import MISSING_ROTATION, edge_ensemble, edge_tuples, with_leaves
from helpers import (assert_scores, labels_of, make_engine, oracle_words, plan_groups, plan_rows, refused, torch_cuda,
                     L)  # noqa: F401 (torch_cuda: a fixture)

HERE = os.path.dirname(os.path.abspath(__file__))
KERNELS = os.path.join(os.path.dirname(HERE), "distributed-decisiontrees_b200", "csrc", "dte_kernels.cuh")

VARIANTS = [E.DTE_KERNEL_GENERIC, E.DTE_KERNEL_TILE, E.DTE_KERNEL_TILE_STAGED, E.DTE_KERNEL_AUTO]
SANITIZER = bool(os.environ.get("DTE_TEST_SANITIZER"))


# ---- the plan table ------------------------------------------------------------------------------------------------
ROWS = plan_rows("plan_table.txt.xz")
NAME_OF = {(r.tune, r.D, r.F, r.C, r.variant): r.name for r in ROWS}


def compiled_templates():
    """Every walk-kernel template the library instantiates (once single-class, once multi-class): the generic kernel
    for both record formats, and each kTileFamilies row for both record formats at its thread bound and, for a bound
    above 384, also at 384 (tile_kernel in dte_device.cuh)."""
    with open(KERNELS) as f:
        src = f.read()
    body = re.search(r"constexpr TileFamily kTileFamilies\[\] = \{(.*?)\};", src, re.S).group(1)
    fams = re.findall(r"\{(\d+), (\d+), (true|false), (\d+)\}", body)
    assert fams, "kTileFamilies not found in dte_kernels.cuh"
    out = {"dt_walk_generic<0>", "dt_walk_generic<1>"}
    for ilp, pair, staged, nt in fams:
        for wide in (0, 1):
            for bound in {int(nt), min(int(nt), 384)}:
                out.add("dt_walk_tile<%s, %s, %d, %d, %d>" % (ilp, pair, staged == "true", wide, bound))
    return out


def matrix_cases():
    """(row, None): the typical and the extreme row of every group on the standard data."""
    out = []
    for (template, C), (typical, extreme) in plan_groups(ROWS).items():
        for kind, row in (("typical", typical), ("extreme", extreme)):
            out.append(pytest.param(row, None, id="%s-C%d-%s-D%d-F%d" % (template.replace(" ", ""), C, kind, row.D, row.F)))
    return out


def edge_cases():
    """(row, missing pattern): the typical row of every group on edge operands (tests/edge_operands.py), the missing
    pattern taken from MISSING_ROTATION by group index."""
    out = []
    for i, ((template, C), (typical, _)) in enumerate(plan_groups(ROWS).items()):
        missing = MISSING_ROTATION[i % len(MISSING_ROTATION)]
        out.append(pytest.param(typical, missing, id="%s-C%d-edge-D%d-F%d-m%08x" % (
            template.replace(" ", ""), C, typical.D, typical.F, missing)))
    return out


# ---- helpers --------------------------------------------------------------------------------------------------------
def tuples(first, n, F, seed, missing_ppm=15000):
    """L.synth_tuples in pieces of ~4 M words, so a wide batch does not hold several full-size temporaries."""
    out = np.empty((n, F), dtype=np.uint32)
    step = max(1, (1 << 22) // F)
    for a in range(0, n, step):
        b = min(n, a + step)
        out[a:b] = L.synth_tuples(first + a, b - a, F, seed=seed, missing_ppm=missing_ppm)
    return out


def ensemble(T, D, F, seed, max_index=None):
    """L.synth_ensemble with one feature index raised to max_index (the engine picks the 64-byte bottom record as soon
    as an index is >= 512).  Default for F > 512: F - 1, so the record format is the one the plan table assumes."""
    W, FI = L.synth_ensemble(T, D, F, seed=seed)
    if max_index is None and F > 512:
        max_index = F - 1
    if max_index is not None:
        FI[0, (1 << D) - 2] = (FI[0, (1 << D) - 2] & 0x2000) | max_index       # the last node of the deepest level
    return W, FI


def check(W, FI, x, D, K, S, C=1, variants=VARIANTS, want=None):
    """Every requested variant on one engine against the oracle; returns (oracle words, {variant: kernel name})."""
    T, F = W.shape[0], x.shape[1]
    wl, fl = L.pack_streams(W, FI, D)
    if want is None:
        want = oracle_words(W, FI, x, D, K, S, C)
    names = {}
    with make_engine(T, D, F, K, S) as e:
        e.load_ensemble(wl, fl, num_classes=C)
        for v in variants:
            e.set_kernel_variant(v)
            names[v] = e.kernel_name()
            sc, lb = e.infer_host(x)
            assert_scores(sc, lb, want, C, "variant %s (%s)" % (E.KERNEL_NAMES[v], names[v]))
    return want, names


def params(name):
    """Template arguments of a kernel name: "dt_walk_tile<4, 2, 1, 0, 384> warps=..." -> [4, 2, 1, 0, 384]."""
    return [int(a) for a in name.split("<")[1].split(">")[0].split(",")]


def assert_table_names(tune, D, F, C, names):
    """Where the geometry is one of the table's, the live kernel names must be the recorded ones."""
    for v, name in names.items():
        key = (tune, D, F, C, v)
        if key in NAME_OF:
            assert name == NAME_OF[key], (key, name)


# ---- 2c: the table on the CPU ---------------------------------------------------------------------------------------
def test_plan_table_reaches_42_kernel_groups():
    """The planner reaches 21 of the 26 walk templates, each single- and multi-class: 42 (template, C) groups, each with
    a typical and an extreme row, and every template it names is one that kTileFamilies instantiates.  A planner change
    that makes another kernel reachable shows up here as a count, not as a kernel no GPU test launches."""
    groups = plan_groups(ROWS)
    assert len(groups) == 42
    compiled = compiled_templates()
    assert len(compiled) == 26                            # x 2 (single-, multi-class) = the 52 walk kernels of libdte.so
    reached = {t for t, _ in groups}
    assert reached <= compiled, reached - compiled
    assert {C for _, C in groups} == {1, 3} and all((t, 1) in groups and (t, 3) in groups for t in reached)
    # the instantiations no plan launches: the non-staged 416-thread builds (that family is capped at 12 warps) and the
    # wide 416-thread builds of the SP = 4 staged families (at F >= 516 at most 3 tuple groups fit)
    assert compiled - reached == {"dt_walk_tile<4, 1, 0, 0, 416>", "dt_walk_tile<4, 1, 0, 1, 416>",
                                  "dt_walk_tile<4, 1, 1, 1, 416>", "dt_walk_tile<4, 2, 1, 1, 416>",
                                  "dt_walk_tile<2, 2, 1, 1, 416>"}
    for (t, C), (typical, extreme) in groups.items():
        for r in (typical, extreme):
            assert r.template == t and r.C == C and r.name.endswith(" classes=3") == (C == 3)
        assert (extreme.D, extreme.F) >= (typical.D, typical.F)
    assert len(matrix_cases()) == 84
    edge = edge_cases()
    assert len(edge) == 42 and {p.values[1] for p in edge} == set(MISSING_ROTATION)


# ---- 2a: the instantiation matrix -----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("row,missing", matrix_cases() + edge_cases())
def test_reachable_instantiation_bit_exact(row, missing, monkeypatch, torch_cuda):
    """The table row's pin, geometry and variant: the live kernel name is the table's, and on enough tuples that every
    CTA walks at least two tiles (ring wrap, tile reload, dead lanes in the last tile) every score word and label equals
    the oracle's, through dte_infer_host and through dte_infer_device on a non-default torch stream.  T is not a
    multiple of 8; C = 3 has classes of 10, 10 and 9 trees (two groups per class).
    Edge cases (missing given): edge operands with that missing pattern on one wave of CTAs plus a ragged tail, the
    same trees loaded with wide and then with small leaves on one handle."""
    torch = torch_cuda
    monkeypatch.setenv("DTE_TUNE", row.tune)
    D, F, C = row.D, row.F, row.C
    T, K, S = (21, 2, 2) if C == 1 else (29, 2, 1)
    if missing is None:
        seed = 5000 + 97 * D + F + C
        W, FI = ensemble(T, D, F, seed)
        loads, missing = [W], L.MISSING_DEFAULT
    else:
        seed = 9000 + 97 * D + F + C
        W, FI, pools = edge_ensemble(T, D, F, seed, leaves="wide", missing=missing)
        loads = [W, with_leaves(W, D, "small", seed)]
    with make_engine(T, D, F, K, S, missing) as e:
        for Wl in loads:
            e.load_ensemble(*L.pack_streams(Wl, FI, D), num_classes=C)
            e.set_kernel_variant(row.variant)
            assert e.kernel_name() == row.name
            info = e.info()
            cap = info["tuples_per_cta"] * info["sm_count"]
            if len(loads) == 1:
                n = cap + 33 if SANITIZER else 2 * cap + 33
                x = tuples(0, n, F, seed + 1)
            else:
                n = cap + 33
                x = edge_tuples(n, F, pools, seed + 1, missing)
            assert cap < n
            want = oracle_words(Wl, FI, x, D, K, S, C, missing)
            sc, lb = e.infer_host(x)
            assert_scores(sc, lb, want, C, "infer_host %s" % row.name)
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                dx = torch.from_numpy(x.view(np.int32)).cuda()
                ds = torch.full(want.shape, float("nan"), dtype=torch.float32, device="cuda")
                dl = torch.full((n,), 77, dtype=torch.uint8, device="cuda")
                e.infer_device(dx, n, ds, dl, stream=st.cuda_stream)
            st.synchronize()
            assert_scores(ds.cpu().numpy(), dl.cpu().numpy(), want, C, "infer_device %s" % row.name)
            del dx, ds, dl


# ---- 2b: edges ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("tune", ["", "pair=2,stages=1"])
def test_depth_14_staged(tune, monkeypatch):
    """D = 14: a 32 KiB tree top in each ring slot.  Shipped pin: dt_walk_tile<4, 1, 1, 0, 416>; pair=2:
    dt_walk_tile<2, 2, 1, 0, 416> (both with phased refill)."""
    monkeypatch.setenv("DTE_TUNE", tune)
    D, F, T = 14, 64, 21
    W, FI = ensemble(T, D, F, seed=5101)
    x = tuples(0, 3001, F, seed=5102, missing_ppm=30000)
    _, names = check(W, FI, x, D, 2, 2, variants=[E.DTE_KERNEL_TILE_STAGED, E.DTE_KERNEL_AUTO])
    assert names[E.DTE_KERNEL_TILE_STAGED].startswith("dt_walk_tile<4, 1, 1, 0, 416>" if not tune else "dt_walk_tile<2, 2, 1, 0, 416>")
    assert "phased=1" in names[E.DTE_KERNEL_TILE_STAGED]
    assert_table_names(tune, D, F, 1, names)


@pytest.mark.gpu
@pytest.mark.parametrize("tune", ["", "ilp=4"])
def test_depth_15_tile_and_generic(tune, monkeypatch):
    """D = 15, the deepest the geometry registers allow: too deep to stage, so the non-staged tile
    (dt_walk_tile<8, 1, 0, 0, 288>, or <4, 1, 0, 0, 384> with ilp=4) and dt_walk_generic<0>."""
    monkeypatch.setenv("DTE_TUNE", tune)
    D, F, T = 15, 32, 13
    W, FI = ensemble(T, D, F, seed=5201)
    x = tuples(0, 2001, F, seed=5202, missing_ppm=30000)
    _, names = check(W, FI, x, D, 2, 1, variants=[E.DTE_KERNEL_TILE, E.DTE_KERNEL_GENERIC, E.DTE_KERNEL_TILE_STAGED])
    assert names[E.DTE_KERNEL_TILE].startswith("dt_walk_tile<8, 1, 0, 0," if not tune else "dt_walk_tile<4, 1, 0, 0,")
    assert names[E.DTE_KERNEL_GENERIC] == "dt_walk_generic<0>"
    assert params(names[E.DTE_KERNEL_TILE_STAGED])[2] == 0              # staged requested, but no ring stage fits
    assert_table_names(tune, D, F, 1, names)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 2])
def test_depth_1_and_2_on_the_tile_kernels(D):
    """D = 1 (extended to two levels) and D = 2: no top levels (Dtop = 0), the whole walk is one bottom record.  The tile
    variants run dt_walk_tile<8, 1, 0, 0, 288> (a staged request falls back to it: nothing to stage)."""
    F, T = 32, 19
    W, FI = ensemble(T, D, F, seed=5300 + D)
    x = tuples(0, 4001, F, seed=5310 + D, missing_ppm=50000)
    _, names = check(W, FI, x, D, 1, 3)
    for v in (E.DTE_KERNEL_TILE, E.DTE_KERNEL_TILE_STAGED, E.DTE_KERNEL_AUTO):
        assert names[v].startswith("dt_walk_tile<8, 1, 0, 0, 288>"), names[v]
    assert_table_names("", D, F, 1, names)


@pytest.mark.gpu
@pytest.mark.parametrize("tune,P", [("pair=1,ilp=8,stages=1", 1), ("pair=2,stages=1", 2), ("pair=4,stages=1", 4)])
def test_tuple_tile_loads(tune, P, monkeypatch):
    """The P warps of a tuple group load alternate 16-feature blocks of the tile and warp 0 of the group loads the
    ragged tail: F = 4 .. 68 covers F/4 below 4, below 4P, not a multiple of 4, and one block per warp plus a tail.
    Staged kernel dt_walk_tile<*, P, 1, 0, *> and the non-staged dt_walk_tile<8, 1, 0, 0, 288>."""
    monkeypatch.setenv("DTE_TUNE", tune)
    D, T = 6, 21
    for F in (4, 8, 12, 20, 36, 52, 68):
        W, FI = ensemble(T, D, F, seed=5400 + F)
        x = tuples(0, 2500 + F, F, seed=5500 + F, missing_ppm=40000)
        _, names = check(W, FI, x, D, 2, 2, variants=[E.DTE_KERNEL_TILE_STAGED, E.DTE_KERNEL_TILE])
        assert re.match(r"dt_walk_tile<\d, %d, 1, 0, " % P, names[E.DTE_KERNEL_TILE_STAGED]), (F, names)
        assert names[E.DTE_KERNEL_TILE].startswith("dt_walk_tile<8, 1, 0, 0,"), (F, names)


@pytest.mark.gpu
@pytest.mark.parametrize("F,max_index,wide", [(512, 511, 0), (1024, 511, 0), (516, 512, 1), (2048, 2047, 1)])
def test_bottom_record_format_edges(F, max_index, wide):
    """The compact 32-byte bottom record packs each node as a 10-bit field (index | missing-right << 9): index 511 with
    the missing-right bit set, at F = 512 and at F = 1024 (every index < 512, so still compact).  Index 512 at F = 516
    needs the 64-byte record; index 2047 at F = 2048 runs dt_walk_generic<1> (no tuple tile fits)."""
    D, T = 8, 21
    rng = np.random.default_rng(F)
    W, FI = L.synth_ensemble(T, D, max_index, seed=5600 + F)          # indexes 0 .. max_index - 1
    hot = rng.random(FI.shape) < 0.3                     # 30 % of the nodes test feature max_index, 2/3 of them go right
    FI[hot] = max_index | np.where(rng.random(int(hot.sum())) < 2 / 3, 0x2000, 0).astype(np.uint16)
    x = tuples(0, 3000, F, seed=5700 + F, missing_ppm=20000)
    x[rng.random(x.shape[0]) < 0.5, max_index] = L.MISSING_DEFAULT
    _, names = check(W, FI, x, D, 2, 2)
    for v, name in names.items():
        if name.startswith("dt_walk_tile<"):
            assert params(name)[3] == wide, name
        else:
            assert name == "dt_walk_generic<%d>" % wide, name
    if F == 2048:
        assert set(names.values()) == {"dt_walk_generic<1>"}
    if wide == (F > 512):                                # the table assumes the wide record exactly when F > 512
        assert_table_names("", D, F, 1, names)


@pytest.mark.gpu
@pytest.mark.parametrize("tune", ["", "pair=4,stages=1", "pair=1,ilp=8,stages=1"])
def test_tuple_count_edges(tune, monkeypatch):
    """n = 1, 31, 33, one tile per SM +- 1, and k tiles + 1 (the last CTA has one live lane), for the shipped plan,
    a P = 4 plan and an ILP = 8 plan, staged and non-staged."""
    monkeypatch.setenv("DTE_TUNE", tune)
    D, F, T, K, S = 10, 128, 21, 2, 2
    W, FI = ensemble(T, D, F, seed=5801)
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F, K, S) as e:
        e.load_ensemble(wl, fl)
        for v in (E.DTE_KERNEL_TILE_STAGED, E.DTE_KERNEL_TILE):
            e.set_kernel_variant(v)
            info = e.info()
            tpc, sm = info["tuples_per_cta"], info["sm_count"]
            ns = sorted({1, 31, 33, tpc * sm - 1, tpc * sm + 1, 3 * tpc + 1, (sm + 1) * tpc + 1})
            x = tuples(0, ns[-1], F, seed=5802, missing_ppm=20000)
            want = oracle_words(W, FI, x, D, K, S, 1)
            for n in ns:
                sc, lb = e.infer_host(x[:n])
                assert_scores(sc, lb, want[:n], 1, "%s n=%d" % (e.kernel_name(), n))


@pytest.mark.gpu
@pytest.mark.parametrize("K,T,S", [(1, 21, 2), (1, 21, 3), (2, 37, 2), (2, 37, 3), (8, 70, 1), (8, 70, 2)])
def test_tree_count_against_slots(K, T, S):
    """S*K*8 tree slots below T (the trees past the last slot are never walked) and above T (whole empty groups add
    exact zeros), K = 1, 2, 8 partials, every variant."""
    D, F = 7, 64
    W, FI = ensemble(T, D, F, seed=5900 + T + S)
    x = tuples(0, 2500, F, seed=5950 + K, missing_ppm=20000)
    check(W, FI, x, D, K, S)


@pytest.mark.gpu
@pytest.mark.parametrize("tune,pref", [("pair=2,ilp=2,stages=2", "dt_walk_tile<2, 2, 1, 0,"), ("pair=4,stages=1", "dt_walk_tile<2, 4, 1, 0,")])
def test_one_group_per_class(tune, pref, monkeypatch, torch_cuda):
    """gpc = 1: C = 10 with T = 75 (8 or 7 trees per class), so a class boundary follows every group — every second
    step with ILP*P = 4 (dt_walk_tile<2, 2, 1>), every step with P = 4 (dt_walk_tile<2, 4, 1>).  Every variant through
    dte_infer_host; the pinned plan also through dte_infer_device_accumulate into zeros (+0 + s = s, exact)."""
    torch = torch_cuda
    monkeypatch.setenv("DTE_TUNE", tune)
    D, F, T, K, S, C = 9, 64, 75, 2, 1, 10
    W, FI = ensemble(T, D, F, seed=6001)
    x = tuples(0, 4001, F, seed=6002, missing_ppm=20000)
    want, names = check(W, FI, x, D, K, S, C)
    assert names[E.DTE_KERNEL_TILE_STAGED].startswith(pref) and names[E.DTE_KERNEL_TILE_STAGED].endswith(" classes=10")
    wl, fl = L.pack_streams(W, FI, D)
    with make_engine(T, D, F, K, S) as e:
        e.load_ensemble(wl, fl, num_classes=C)
        e.set_kernel_variant(E.DTE_KERNEL_TILE_STAGED)
        dx = torch.from_numpy(x.view(np.int32)).cuda()
        acc = torch.zeros((x.shape[0], C), dtype=torch.float32, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        e.infer_device_accumulate(dx, x.shape[0], acc, stream=st)
        torch.cuda.synchronize()
        assert_scores(acc.cpu().numpy(), None, want, C, "accumulate %s" % e.kernel_name())


@pytest.mark.gpu
def test_classes_without_trees():
    """C = 5 with T = 3: classes 3 and 4 hold no tree and score +0 (the all-zero word) on every kernel; every leaf of
    classes 0..2 is negative, so the first class of maximal score is 3 for every tuple."""
    D, F, T, C = 6, 32, 3, 5
    W, FI = ensemble(T, D, F, seed=6101)
    n_int = (1 << D) - 1
    u = W[:, n_int:].view(np.float32)
    W[:, n_int:] = (-(np.abs(u) + np.float32(0.125))).astype(np.float32).view(np.uint32)
    x = tuples(0, 3001, F, seed=6102, missing_ppm=20000)
    want, _ = check(W, FI, x, D, 1, 1, C)
    assert (want[:, 3:] == 0).all() and (want[:, :3].view(np.float32) < 0).all()
    assert (labels_of(want, C) == 3).all()


@pytest.mark.gpu
def test_256_classes():
    """C = 256, the most a one-byte label holds, with T = 300 (2 trees in classes 0..43, 1 in the rest); the leaves of
    tree 255 are scaled up so that label 255 wins on part of the tuples."""
    D, F, T, C = 5, 32, 300, 256
    W, FI = ensemble(T, D, F, seed=6201)
    n_int = (1 << D) - 1
    W[255, n_int:] = (W[255, n_int:].view(np.float32) * np.float32(4096.0)).view(np.uint32)
    x = tuples(0, 2000, F, seed=6202, missing_ppm=20000)
    want, names = check(W, FI, x, D, 1, 1, C)
    lab = labels_of(want, C)
    assert (lab == 255).any() and (lab != 255).any()
    assert all(n.endswith(" classes=256") for n in names.values())


@pytest.mark.gpu
@pytest.mark.parametrize("tune,stages,phased", [("fill=1,phased=0", None, 0), ("phased=2", None, 1), ("phased=3", None, 1),
                                                ("ilp=4,pair=1,stages=3", 3, 1), ("ilp=2,pair=2,stages=4", 4, 1)])
def test_ring_fill_knobs(tune, stages, phased, monkeypatch):
    """Staged D = 12 walk (8 KiB tree tops) under the ring-fill knobs: one bulk copy per tree (fill=1, which applies
    when phased refill is off), phased refill with part A ending one or two levels earlier (phased=2, 3), and three- and
    four-stage rings.  The kernel name shows the stage count and whether phased refill is on."""
    monkeypatch.setenv("DTE_TUNE", tune)
    D, F, T, K, S = 12, 256, 21, 8, 1
    W, FI = ensemble(T, D, F, seed=6301)
    with make_engine(T, D, F, K, S) as e:
        e.load_ensemble(*L.pack_streams(W, FI, D))
        e.set_kernel_variant(E.DTE_KERNEL_TILE_STAGED)
        info = e.info()
        n = info["tuples_per_cta"] * info["sm_count"] * (1 if SANITIZER else 2) + 33
    x = tuples(0, n, F, seed=6302, missing_ppm=20000)
    _, names = check(W, FI, x, D, K, S, variants=[E.DTE_KERNEL_TILE_STAGED])
    name = names[E.DTE_KERNEL_TILE_STAGED]
    assert re.match(r"dt_walk_tile<\d, \d, 1, 0, ", name), name
    assert "phased=%d" % phased in name, name
    if stages:
        assert " stages=%d " % stages in name, name


@pytest.mark.gpu
def test_misaligned_device_pointers_are_refused(torch_cuda):
    """dte_infer_device and dte_infer_device_accumulate refuse a tuple pointer that is not 16-byte aligned (the tile
    kernels read rows as 128-bit vectors) and a score pointer that is not 4-byte aligned, with DTE_ERR_ARG and before
    any launch; a correct call on the same engine afterwards returns the oracle's words (no sticky CUDA error)."""
    torch = torch_cuda
    D, F, T, K, S, n = 8, 64, 21, 2, 2, 1000
    W, FI = ensemble(T, D, F, seed=6401)
    x = tuples(0, n, F, seed=6402)
    want = oracle_words(W, FI, x, D, K, S, 1)
    st = torch.cuda.current_stream().cuda_stream
    with make_engine(T, D, F, K, S) as e:
        e.load_ensemble(*L.pack_streams(W, FI, D))
        dx = torch.zeros(n * F + 8, dtype=torch.int32, device="cuda")
        dx[: n * F] = torch.from_numpy(x.view(np.int32).ravel()).cuda()
        ds = torch.zeros(n + 4, dtype=torch.float32, device="cuda")
        for v in VARIANTS:
            e.set_kernel_variant(v)
            for call in (lambda t, s: e.infer_device(t, n, s, None, stream=st),
                         lambda t, s: e.infer_device_accumulate(t, n, s, stream=st)):
                refused(lambda: call(dx.data_ptr() + 4, ds.data_ptr()), E.DTE_ERR_ARG, "d_tuples not 16-byte aligned")
                refused(lambda: call(dx.data_ptr(), ds.data_ptr() + 2), E.DTE_ERR_ARG, "not 4-byte aligned")
        torch.cuda.synchronize()
        for v in VARIANTS:
            e.set_kernel_variant(v)
            out = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
            e.infer_device(dx, n, out, None, stream=st)
            torch.cuda.synchronize()
            assert_scores(out.cpu().numpy(), None, want, 1, "aligned call after refusals, %s" % e.kernel_name())


@pytest.mark.gpu
@pytest.mark.parametrize("F", [2048, 1796])
def test_tuple_offsets_beyond_4_gib(F, torch_cuda):
    """A tuple buffer of a little over 4 GiB filled on the device by dte_synth_tuples_device: F = 2048 runs
    dt_walk_generic<1>, F = 1796 the widest tile plan (one tuple group per CTA, 64-byte records).  The first 256 and
    the last 512 tuples, whose byte offsets pass 2^32, equal the oracle's scores of the same tuples made on the host."""
    torch = torch_cuda
    free, _ = torch.cuda.mem_get_info()
    if free < 6 << 30:
        pytest.skip("needs 6 GiB of free device memory, %.1f GiB free" % (free / 2 ** 30))
    D, T, K, S, seed = 6, 21, 2, 2, 0x4B1D
    n = (4 << 30) // (4 * F) + 1024
    assert (n - 512) * F * 4 >= 1 << 32
    W, FI = ensemble(T, D, F, seed=6500 + F)
    wl, fl = L.pack_streams(W, FI, D)
    st = torch.cuda.current_stream().cuda_stream
    with make_engine(T, D, F, K, S) as e:
        e.load_ensemble(wl, fl)
        name = e.kernel_name()
        assert name == NAME_OF[("", D, F, 1, E.DTE_KERNEL_AUTO)]
        if F == 2048:
            assert name == "dt_walk_generic<1>"
        else:
            assert name.startswith("dt_walk_tile<") and params(name)[3] == 1, name
        dx = torch.empty((n, F), dtype=torch.int32, device="cuda")
        ds = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
        try:
            e.synth_tuples_device(dx, 0, n, F, seed, 15000, L.MISSING_DEFAULT, stream=st)
            e.infer_device(dx, n, ds, None, stream=st)
            torch.cuda.synchronize()
            got = ds.cpu().numpy().view(np.uint32)
        finally:
            del dx, ds
            torch.cuda.empty_cache()
    for first, count in ((0, 256), (n - 512, 512)):
        x = L.synth_tuples(first, count, F, seed=seed, missing_ppm=15000)
        want = oracle_words(W, FI, x, D, K, S, 1)
        assert_scores(got[first:first + count], None, want, 1, "%s tuples %d..%d" % (name, first, first + count))
