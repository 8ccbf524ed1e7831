"""Every refusal of a walk kind that needs no kernel to provoke, pinned with its status code and its full message: the
layout the kind reads is not resident, a misaligned device pointer, an attribution call on an ensemble-sharded handle,
a multi-class run whose slots hold fewer trees than its largest class, and an interaction row over 2^24 words.  Each of
the seven kinds runs on a single-device handle and on a [0, 0, 0] ensemble-sharded handle (three ring positions sharing
one GPU).  Device calls that are to be refused walk no tuples (n = 0), so nothing runs whatever the engine decides."""
import numpy as np
import pytest

import ddt_b200 as ddt
from ddt_b200 import engine as E
from helpers import make_engine, multi_node_regs, refused_exactly, torch_cuda, write_regs, L  # noqa: F401

pytestmark = pytest.mark.gpu

T, D, F, K, n = 40, 5, 32, 2, 8

# the suffix of each kind's calls: infer_host<sfx>, infer_device<sfx>, kernel_name<sfx>
KINDS = ["", "_binned", "_leaves", "_contribs", "_interactions", "_approx_contribs", "_interventional"]
ATTRIBUTION = {"_contribs": "contributions", "_interactions": "interaction values", "_approx_contribs": "contributions",
               "_interventional": "contributions"}
NO_ENSEMBLE = "no ensemble loaded"
MISSING = {
    "": NO_ENSEMBLE,
    "_binned": "no binned layout resident: load the ensemble with dte_load_ensemble_binned",
    "_leaves": "no leaf-id layout resident: place the ensemble with DTE_OPT_LEAF_LAYOUT = 1",
    "_contribs": "no contribution layout resident: load the ensemble with dte_load_ensemble_contribs",
    "_interactions": "no contribution layout resident: load the ensemble with dte_load_ensemble_contribs",
    "_approx_contribs": "no approximate-contribution table resident: load the ensemble with dte_load_ensemble_approx_contribs",
    "_interventional": "no interventional layout resident: load the ensemble with dte_load_ensemble_interventional",
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
    "_interventional": ("dte_infer_device_interventional: d_tuples not 16-byte aligned",
                        "dte_infer_device_interventional: d_contribs not 4-byte aligned"),
}
SHARDED = ("infer_host%s: an ensemble-sharded handle cannot return %s; use a single-device or data-sharded handle")
SLOTS = ("reg 205: S=1 x K=2 x 8 slots hold fewer trees than the largest of the 2 classes (20 trees): a multi-class run "
         "needs S >= 2")


@pytest.fixture(scope="module")
def case():
    W, FI = L.synth_ensemble(T, D, F, seed=5101, cuts=16)     # binnable: 16 cuts per feature
    wl, fl = L.pack_streams(W, FI, D)
    cov = L.synth_covers(FI, D, seed=5102)
    x = L.synth_tuples(0, n, F, seed=5103)
    bg = L.synth_tuples(0, 3, F, seed=5104)
    return wl, fl, cov, bg, x


def sharded():
    e = ddt.Engine([0, 0, 0])
    write_regs(e, multi_node_regs(T, D, F, K, n, 3, "ensemble"))
    return e


def load(e, sfx, wl, fl, cov, bg, **kw):
    """Load the ensemble with the layout the kind reads."""
    extra = {"_binned": dict(binned=True), "_leaves": dict(leaves=True), "_contribs": dict(covers=cov),
             "_interactions": dict(covers=cov), "_approx_contribs": dict(covers=cov, approx=True),
             "_interventional": dict(background=bg)}.get(sfx, {})
    e.load_ensemble(wl, fl, **extra, **kw)


def host(e, sfx, x):
    return lambda: getattr(e, "infer_host" + sfx)(np.zeros((n, F), np.uint8) if sfx == "_binned" else x)


def device(e, sfx, d_in=None, d_out=None):
    return lambda: getattr(e, "infer_device" + sfx)(d_in, 0, d_out)


def name(e, sfx):
    return getattr(e, "kernel_name" + sfx)


@pytest.mark.parametrize("sfx", KINDS, ids=lambda s: s[1:] or "fp32")
def test_missing_layout_single(torch_cuda, case, sfx):
    """No ensemble: every infer call says so, the name call names the kind's layout; a plain load: every call of
    another kind names the layout it reads."""
    wl, fl, cov, bg, x = case
    with make_engine(T, D, F, K, 1) as e:
        refused_exactly(host(e, sfx, x), E.DTE_ERR_STATE, NO_ENSEMBLE)
        refused_exactly(device(e, sfx), E.DTE_ERR_STATE, NO_ENSEMBLE)
        refused_exactly(name(e, sfx), E.DTE_ERR_STATE, MISSING[sfx])
        if sfx:
            e.load_ensemble(wl, fl)
            for call in (host(e, sfx, x), device(e, sfx), name(e, sfx)):
                refused_exactly(call, E.DTE_ERR_STATE, MISSING[sfx])


@pytest.mark.parametrize("sfx", KINDS, ids=lambda s: s[1:] or "fp32")
def test_missing_layout_and_attribution_sharded(torch_cuda, case, sfx):
    """An ensemble-sharded handle refuses the attribution host calls before it looks for a layout, with or without
    one; the other kinds and every name call name the missing layout as a single-device handle does."""
    wl, fl, cov, bg, x = case
    with sharded() as e:
        sharded_msg = SHARDED % (sfx, ATTRIBUTION[sfx]) if sfx in ATTRIBUTION else None
        if sharded_msg:
            refused_exactly(host(e, sfx, x), E.DTE_ERR_CONFIG, sharded_msg)
        else:
            refused_exactly(host(e, sfx, x), E.DTE_ERR_STATE, NO_ENSEMBLE)
        refused_exactly(name(e, sfx), E.DTE_ERR_STATE, MISSING[sfx])
        if not sfx:
            return
        e.load_ensemble(wl, fl)
        if sharded_msg:
            refused_exactly(host(e, sfx, x), E.DTE_ERR_CONFIG, sharded_msg)
        else:
            refused_exactly(host(e, sfx, x), E.DTE_ERR_STATE, MISSING[sfx])
        refused_exactly(name(e, sfx), E.DTE_ERR_STATE, MISSING[sfx])
        if sharded_msg:
            load(e, sfx, wl, fl, cov, bg)
            refused_exactly(host(e, sfx, x), E.DTE_ERR_CONFIG, sharded_msg)


@pytest.mark.parametrize("sfx", KINDS, ids=lambda s: s[1:] or "fp32")
def test_misaligned_device_pointers(torch_cuda, case, sfx):
    """The input must be 16-byte aligned, the output 4-byte (leaf cells: 16-byte), whatever is resident."""
    wl, fl, cov, bg, _ = case
    buf = torch_cuda.zeros(1024, dtype=torch_cuda.int32, device="cuda")
    base = buf.data_ptr()
    bad_out = base + (8 if sfx == "_leaves" else 2)
    want_in, want_out = MISALIGNED[sfx]
    with make_engine(T, D, F, K, 1) as e:
        for loaded in (False, True):
            if loaded:
                load(e, sfx, wl, fl, cov, bg)
            refused_exactly(device(e, sfx, base + 4, base), E.DTE_ERR_ARG, want_in)
            refused_exactly(device(e, sfx, base, bad_out), E.DTE_ERR_ARG, want_out)
            if not sfx:
                refused_exactly(lambda: e.infer_device_accumulate(base + 4, 0, base), E.DTE_ERR_ARG,
                                "dte_infer_device_accumulate: d_tuples not 16-byte aligned")
                refused_exactly(lambda: e.infer_device_accumulate(base, 0, base + 2), E.DTE_ERR_ARG,
                                "dte_infer_device_accumulate: d_scores_accum not 4-byte aligned")


@pytest.mark.parametrize("sfx", KINDS, ids=lambda s: s[1:] or "fp32")
def test_multi_class_slots(torch_cuda, case, sfx):
    """S = 1, K = 2: 16 slots for 20 trees per class.  Every kind but the leaf walk, which walks every tree whatever K
    and S say, refuses the run."""
    wl, fl, cov, bg, x = case
    with make_engine(T, D, F, K, 1) as e:
        load(e, sfx, wl, fl, cov, bg, num_classes=2)
        if sfx == "_leaves":
            assert e.infer_host_leaves(x).shape == (n, T)
            return
        refused_exactly(host(e, sfx, x), E.DTE_ERR_CONFIG, SLOTS)
        refused_exactly(device(e, sfx), E.DTE_ERR_CONFIG, SLOTS)


def test_interaction_row_cap(torch_cuda):
    """C = 4, F = 2048: 4 x 2049^2 words of one tuple's interaction row exceed 2^24."""
    Dw, Fw = 2, 2048
    W, FI = L.synth_ensemble(8, Dw, Fw, seed=5111)
    cov = L.synth_covers(FI, Dw, seed=5112)
    wl, fl = L.pack_streams(W, FI, Dw)
    x = L.synth_tuples(0, 2, Fw, seed=5113)
    msg = "an interaction row of 4 classes x 2049 x 2049 words exceeds 64 MiB (2^24 words)"
    with make_engine(8, Dw, Fw, 8, 1) as e:
        e.load_ensemble(wl, fl, num_classes=4, covers=cov)
        refused_exactly(lambda: e.infer_host_interactions(x), E.DTE_ERR_UNSUPPORTED, msg)
        refused_exactly(lambda: e.infer_device_interactions(None, 0, None), E.DTE_ERR_UNSUPPORTED, msg)


# Every row of the load table: the load, the kinds whose layouts it leaves resident (the leaf ids too when `leaves`), and
# a refusal of the same load kind, which must leave whatever the previous row placed as it was.
# ensemble_bytes of each row (T = 40, D = 5, F = 32, three background rows), without and with the leaf ids
BYTES = {
    ("none", False): 0, ("none", True): 0,
    ("plain", False): 14720, ("plain", True): 24960,
    ("classes", False): 17664, ("classes", True): 29952,
    ("binned", False): 26240, ("binned", True): 36480,
    ("contribs", False): 188816, ("contribs", True): 199056,
    ("approx", False): 48000, ("approx", True): 48000,
    ("interventional", False): 86800, ("interventional", True): 97040,
    ("stream", False): 14720, ("stream", True): 24960,
}


def test_resident_layouts_per_load(torch_cuda, case):
    """Each load answers the kernel-name calls of exactly the kinds whose layouts it builds; every other call names the
    layout it misses.  A refused load changes nothing resident.  The tree line stream places the base pack alone."""
    wl, fl, cov, bg, x = case
    W, FI = L.unpack_streams(wl, fl, D)
    FI_wide = FI.copy()
    FI_wide[0, 0] = (FI_wide[0, 0] & ~np.uint16(0x7FF)) | np.uint16(F)
    wl_wide, fl_wide = L.pack_streams(W, FI_wide, D)
    Wr, _ = L.synth_ensemble(T, D, F, seed=5105)               # thresholds drawn freely: all on feature 0
    wl_many, fl_many = L.pack_streams(Wr, FI & np.uint16(0x2000), D)
    n_edges = len(np.unique(Wr[:, :(1 << D) - 1]))
    cov_bad = cov.copy()
    cov_bad[0, 0] = 0
    bad_cover = "covers: tree 0 cell 0 has cover 0: a live node or reachable leaf needs a finite cover > 0"

    def null_background(e):
        e._check(e._lib.dte_load_ensemble_interventional(e._h, E._ptr(wl), wl.nbytes // 16, E._ptr(fl), fl.nbytes // 16,
                                                         0, 0, 1, None, 0))

    rows = [
        ("plain", dict(), {""},
         (lambda e: e.load_ensemble(wl_wide, fl_wide), E.DTE_ERR_UNSUPPORTED, "tree 0 node 0: feature index 32 >= 32 features")),
        ("classes", dict(num_classes=2), {""},
         (lambda e: e.load_ensemble(wl, fl, num_classes=257), E.DTE_ERR_ARG, "num_classes = 257, need 1..256")),
        ("binned", dict(binned=True), {"", "_binned"},
         (lambda e: e.load_ensemble(wl_many, fl_many, binned=True), E.DTE_ERR_UNSUPPORTED,
          "feature 0 has %d distinct thresholds: a binned layout holds at most 254 per feature" % n_edges)),
        ("contribs", dict(covers=cov), {"", "_contribs", "_interactions"},
         (lambda e: e.load_ensemble(wl, fl, covers=cov_bad), E.DTE_ERR_ARG, bad_cover)),
        ("approx", dict(covers=cov, approx=True), {"", "_approx_contribs", "_leaves"},
         (lambda e: e.load_ensemble(wl, fl, covers=cov_bad, approx=True), E.DTE_ERR_ARG, bad_cover)),
        ("interventional", dict(background=bg), {"", "_interventional"},
         (null_background, E.DTE_ERR_ARG, "dte_load_ensemble_interventional: background is NULL")),
    ]

    def check(e, answers, key):
        for sfx in KINDS:
            if sfx in answers:
                assert isinstance(name(e, sfx)(), str), (key, sfx)
            else:
                refused_exactly(name(e, sfx), E.DTE_ERR_STATE, MISSING[sfx])
        assert e.info()["ensemble_bytes"] == BYTES[key], key

    for leaves in (False, True):
        with make_engine(T, D, F, K, 1) as e:
            answers, key = set(), ("none", leaves)
            for row, kw, builds, (bad_load, code, msg) in rows:
                refused_exactly(lambda: bad_load(e), code, msg)
                check(e, answers, key)
                e.load_ensemble(wl, fl, leaves=leaves, **kw)
                answers, key = builds | ({"_leaves"} if leaves else set()), (row, leaves)
                check(e, answers, key)
            e.configure(T, D, 4 * F, clusters=K, n_tuples=n)
            e.set_option(E.DTE_OPT_LEAF_LAYOUT, int(leaves))
            e.start()
            e.stream_write(wl)
            e.stream_write(fl)
            e.stream_write(x)
            e.stream_flush()
            check(e, {"", "_leaves"} if leaves else {""}, ("stream", leaves))
