"""Every refusal of a walk kind that needs no kernel to provoke, pinned with its status code and its full message: the
layout the kind reads is not resident, a misaligned device pointer, an attribution call on an ensemble-sharded handle,
a multi-class run whose slots hold fewer trees than its largest class, and an interaction row over 2^24 words.  Each of
the six kinds runs on a single-device handle and on a [0, 0, 0] ensemble-sharded handle (three ring positions sharing
one GPU).  Device calls that are to be refused walk no tuples (n = 0), so nothing runs whatever the engine decides."""
import numpy as np
import pytest

import ddt_b200 as ddt
from ddt_b200 import engine as E
from helpers import geometry_regs, multi_node_regs, L

pytestmark = pytest.mark.gpu

DTE_ERR_ARG, DTE_ERR_STATE, DTE_ERR_CONFIG, DTE_ERR_UNSUPPORTED = -1, -2, -3, -4
T, D, F, K, n = 40, 5, 32, 2, 8

# the suffix of each kind's calls: infer_host<sfx>, infer_device<sfx>, kernel_name<sfx>
KINDS = ["", "_binned", "_leaves", "_contribs", "_interactions", "_approx_contribs"]
ATTRIBUTION = {"_contribs": "contributions", "_interactions": "interaction values", "_approx_contribs": "contributions"}
NO_ENSEMBLE = "no ensemble loaded"
MISSING = {
    "": NO_ENSEMBLE,
    "_binned": "no binned layout resident: load the ensemble with dte_load_ensemble_binned",
    "_leaves": "no leaf-id layout resident: place the ensemble with DTE_OPT_LEAF_LAYOUT = 1",
    "_contribs": "no contribution layout resident: load the ensemble with dte_load_ensemble_contribs",
    "_interactions": "no contribution layout resident: load the ensemble with dte_load_ensemble_contribs",
    "_approx_contribs": "no approximate-contribution table resident: load the ensemble with dte_load_ensemble_approx_contribs",
}
MISALIGNED = {                   # (input, output) refusals of dte_infer_device<sfx>
    "": ("dte_infer_device: d_tuples not 16-byte aligned", "dte_infer_device: d_scores not 4-byte aligned"),
    "_binned": ("dte_infer_device_binned: d_bins not 16-byte aligned", "dte_infer_device_binned: d_scores not 4-byte aligned"),
    "_leaves": ("dte_infer_device_leaves: d_tuples not 16-byte aligned", "dte_infer_device_leaves: d_leaves not 16-byte aligned"),
    "_contribs": ("dte_infer_device_contribs: d_tuples not 16-byte aligned",
                  "dte_infer_device_contribs: d_contribs not 4-byte aligned"),
    "_interactions": ("dte_infer_device_interactions: d_tuples not 16-byte aligned",
                      "dte_infer_device_interactions: d_inter not 4-byte aligned"),
    "_approx_contribs": ("dte_infer_device_approx_contribs: d_tuples not 16-byte aligned",
                         "dte_infer_device_approx_contribs: d_contribs not 4-byte aligned"),
}
SHARDED = ("infer_host%s: an ensemble-sharded handle cannot return %s; use a single-device or data-sharded handle")
SLOTS = ("reg 205: S=1 x K=2 x 8 slots hold fewer trees than the largest of the 2 classes (20 trees): a multi-class run "
         "needs S >= 2")


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    assert torch.cuda.is_available(), "these tests need the H100"
    return torch


@pytest.fixture(scope="module")
def case():
    W, FI = L.synth_ensemble(T, D, F, seed=5101, cuts=16)     # binnable: 16 cuts per feature
    wl, fl = L.pack_streams(W, FI, D)
    cov = L.synth_covers(FI, D, seed=5102)
    x = L.synth_tuples(0, n, F, seed=5103)
    return wl, fl, cov, x


def single(S=1):
    e = ddt.Engine(0)
    for a, v in sorted(geometry_regs(T, D, F, K, S, L.MISSING_DEFAULT).items()):
        e.softreg_write(a, v)
    return e


def sharded():
    e = ddt.Engine([0, 0, 0])
    for a, v in sorted(multi_node_regs(T, D, F, K, n, 3, "ensemble").items()):
        e.softreg_write(a, v)
    return e


def load(e, sfx, wl, fl, cov, **kw):
    """Load the ensemble with the layout the kind reads."""
    extra = {"_binned": dict(binned=True), "_leaves": dict(leaves=True), "_contribs": dict(covers=cov),
             "_interactions": dict(covers=cov), "_approx_contribs": dict(covers=cov, approx=True)}.get(sfx, {})
    e.load_ensemble(wl, fl, **extra, **kw)


def host(e, sfx, x):
    return lambda: getattr(e, "infer_host" + sfx)(np.zeros((n, F), np.uint8) if sfx == "_binned" else x)


def device(e, sfx, d_in=None, d_out=None):
    return lambda: getattr(e, "infer_device" + sfx)(d_in, 0, d_out)


def name(e, sfx):
    return getattr(e, "kernel_name" + sfx)


def refused(call, code, msg):
    with pytest.raises(E.DteError) as ei:
        call()
    assert ei.value.code == code, str(ei.value)
    assert str(ei.value) == "dte error %d: %s" % (code, msg)


@pytest.mark.parametrize("sfx", KINDS, ids=lambda s: s[1:] or "fp32")
def test_missing_layout_single(torch_cuda, case, sfx):
    """No ensemble: every infer call says so, the name call names the kind's layout; a plain load: every call of
    another kind names the layout it reads."""
    wl, fl, cov, x = case
    with single() as e:
        refused(host(e, sfx, x), DTE_ERR_STATE, NO_ENSEMBLE)
        refused(device(e, sfx), DTE_ERR_STATE, NO_ENSEMBLE)
        refused(name(e, sfx), DTE_ERR_STATE, MISSING[sfx])
        if sfx:
            e.load_ensemble(wl, fl)
            for call in (host(e, sfx, x), device(e, sfx), name(e, sfx)):
                refused(call, DTE_ERR_STATE, MISSING[sfx])


@pytest.mark.parametrize("sfx", KINDS, ids=lambda s: s[1:] or "fp32")
def test_missing_layout_and_attribution_sharded(torch_cuda, case, sfx):
    """An ensemble-sharded handle refuses the attribution host calls before it looks for a layout, with or without
    one; the other kinds and every name call name the missing layout as a single-device handle does."""
    wl, fl, cov, x = case
    with sharded() as e:
        sharded_msg = SHARDED % (sfx, ATTRIBUTION[sfx]) if sfx in ATTRIBUTION else None
        if sharded_msg:
            refused(host(e, sfx, x), DTE_ERR_CONFIG, sharded_msg)
        else:
            refused(host(e, sfx, x), DTE_ERR_STATE, NO_ENSEMBLE)
        refused(name(e, sfx), DTE_ERR_STATE, MISSING[sfx])
        if not sfx:
            return
        e.load_ensemble(wl, fl)
        if sharded_msg:
            refused(host(e, sfx, x), DTE_ERR_CONFIG, sharded_msg)
        else:
            refused(host(e, sfx, x), DTE_ERR_STATE, MISSING[sfx])
        refused(name(e, sfx), DTE_ERR_STATE, MISSING[sfx])
        if sharded_msg:
            load(e, sfx, wl, fl, cov)
            refused(host(e, sfx, x), DTE_ERR_CONFIG, sharded_msg)


@pytest.mark.parametrize("sfx", KINDS, ids=lambda s: s[1:] or "fp32")
def test_misaligned_device_pointers(torch_cuda, case, sfx):
    """The input must be 16-byte aligned, the output 4-byte (leaf cells: 16-byte), whatever is resident."""
    wl, fl, cov, _ = case
    buf = torch_cuda.zeros(1024, dtype=torch_cuda.int32, device="cuda")
    base = buf.data_ptr()
    bad_out = base + (8 if sfx == "_leaves" else 2)
    want_in, want_out = MISALIGNED[sfx]
    with single() as e:
        for loaded in (False, True):
            if loaded:
                load(e, sfx, wl, fl, cov)
            refused(device(e, sfx, base + 4, base), DTE_ERR_ARG, want_in)
            refused(device(e, sfx, base, bad_out), DTE_ERR_ARG, want_out)
            if not sfx:
                refused(lambda: e.infer_device_accumulate(base + 4, 0, base), DTE_ERR_ARG,
                        "dte_infer_device_accumulate: d_tuples not 16-byte aligned")
                refused(lambda: e.infer_device_accumulate(base, 0, base + 2), DTE_ERR_ARG,
                        "dte_infer_device_accumulate: d_scores_accum not 4-byte aligned")


@pytest.mark.parametrize("sfx", KINDS, ids=lambda s: s[1:] or "fp32")
def test_multi_class_slots(torch_cuda, case, sfx):
    """S = 1, K = 2: 16 slots for 20 trees per class.  Every kind but the leaf walk, which walks every tree whatever K
    and S say, refuses the run."""
    wl, fl, cov, x = case
    with single(S=1) as e:
        load(e, sfx, wl, fl, cov, num_classes=2)
        if sfx == "_leaves":
            assert e.infer_host_leaves(x).shape == (n, T)
            return
        refused(host(e, sfx, x), DTE_ERR_CONFIG, SLOTS)
        refused(device(e, sfx), DTE_ERR_CONFIG, SLOTS)


def test_interaction_row_cap(torch_cuda):
    """C = 4, F = 2048: 4 x 2049^2 words of one tuple's interaction row exceed 2^24."""
    Dw, Fw = 2, 2048
    W, FI = L.synth_ensemble(8, Dw, Fw, seed=5111)
    cov = L.synth_covers(FI, Dw, seed=5112)
    wl, fl = L.pack_streams(W, FI, Dw)
    x = L.synth_tuples(0, 2, Fw, seed=5113)
    msg = "an interaction row of 4 classes x 2049 x 2049 words exceeds 64 MiB (2^24 words)"
    with ddt.Engine(0) as e:
        for a, v in sorted(geometry_regs(8, Dw, Fw, 8, 1, L.MISSING_DEFAULT).items()):
            e.softreg_write(a, v)
        e.load_ensemble(wl, fl, num_classes=4, covers=cov)
        refused(lambda: e.infer_host_interactions(x), DTE_ERR_UNSUPPORTED, msg)
        refused(lambda: e.infer_device_interactions(None, 0, None), DTE_ERR_UNSUPPORTED, msg)
