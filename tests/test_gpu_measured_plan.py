"""The launch plan a large-workload handle measures at load: whichever plan wins, the walk returns the static plan's words.

A single-device handle configured for >= 8 M tuples (reg 207) times the staged candidates when it loads the ensemble
and keeps the fastest if it beats the built-in plan by 2 %.  The plan only changes how the walk is launched, so every
score word and label must equal those of a handle on the built-in plan, and the oracle's."""
import numpy as np
import pytest

import ddt_b200 as ddt
from ddt_b200 import engine as E
from oracle import oracle as O

pytestmark = pytest.mark.gpu

L = ddt.layout
T, D, F, K = 1024, 12, 256, 8          # cfg3
S = -(-T // (8 * K))
N = 1 << 20


def test_measured_plan_at_cfg3_is_bit_exact_with_the_static_plan():
    import torch
    assert torch.cuda.is_available(), "this test needs the H100"
    W, FI = L.synth_ensemble(T, D, F)
    wl, fl = L.pack_streams(W, FI, D)
    with ddt.Engine(0) as big, ddt.Engine(0) as small:
        big.configure(T, D, 4 * F, clusters=K, missing_value=L.MISSING_DEFAULT, n_tuples=50_000_000)
        big.load_ensemble(wl, fl)
        small.configure(T, D, 4 * F, clusters=K, missing_value=L.MISSING_DEFAULT, n_tuples=N)
        small.load_ensemble(wl, fl)
        info = big.info()
        assert info["plan_source"] in ("static", "measured"), info
        assert small.info()["plan_source"] == "static"
        name = big.kernel_name()
        assert name.startswith("dt_walk_tile<") and "stages=" in name, name
        assert (info["plan_source"] == "static") == (name == small.kernel_name()), (name, small.kernel_name())

        d_x = torch.empty((N, F), dtype=torch.int32, device="cuda")
        small.synth_tuples_device(d_x, 0, N, F, 0x7091E5, 10000, L.MISSING_DEFAULT)
        s_big, s_small = (torch.empty(N, dtype=torch.float32, device="cuda") for _ in range(2))
        l_big, l_small = (torch.empty(N, dtype=torch.uint8, device="cuda") for _ in range(2))
        big.infer_device(d_x, N, s_big, l_big)
        small.infer_device(d_x, N, s_small, l_small)
        torch.cuda.synchronize()
        assert torch.equal(s_big.view(torch.int32), s_small.view(torch.int32)), name
        assert torch.equal(l_big, l_small), name

        idx = np.unique(np.random.default_rng(3).choice(N, 4096, replace=False))
        sel = torch.from_numpy(idx).cuda()
        xs = d_x[sel].cpu().numpy().view(np.uint32)
        w_cls, f_cls = L.tree_cls(D)
        want = O.scores_blocked(O.make_cfg(D, K, S, L.MISSING_DEFAULT, w_cls, f_cls, F // 4, T), wl, fl, xs,
                                threads=O.max_threads())
        got = s_big[sel].cpu().numpy().view(np.uint32)
        assert idx.size == 4096 and (got == want).all(), "%d/4096 words differ (%s)" % ((got != want).sum(), name)
        assert (l_big[sel].cpu().numpy() == O.labels(want)).all()

        # a forced variant runs the static plans; AUTO returns to the measured one
        big.set_kernel_variant(E.DTE_KERNEL_TILE)
        small.set_kernel_variant(E.DTE_KERNEL_TILE)
        assert big.kernel_name() == small.kernel_name() and big.info()["plan_source"] == "static"
        big.set_kernel_variant(E.DTE_KERNEL_AUTO)
        assert big.kernel_name() == name and big.info()["plan_source"] == info["plan_source"]
