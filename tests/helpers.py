"""Shared test helpers: build streams/config for a case, run the oracle on it, and drive and check an engine.

Importing this module needs no GPU: torch is imported only when the `torch_cuda` fixture runs."""
import collections
import lzma
import os

import numpy as np
import pytest

import ddt_b200 as ddt
from ddt_b200 import engine as E
from oracle import oracle as O

L = ddt.layout
HERE = os.path.dirname(os.path.abspath(__file__))
CANARY = 0x7A7A7A7A            # the word device_rows leaves after the last row


def kat_arrays(case):
    """KAT case -> (W uint32 [T, 2^(D+1)-1], FI uint16 [T, 2^D-1], tuples uint32 [n, F])."""
    W = np.array([t["W"] for t in case["trees"]], dtype=np.uint32)
    FI = np.array([t["FI"] for t in case["trees"]], dtype=np.uint16)
    x = np.array(case["tuples"], dtype=np.uint32)
    return W, FI, x


def oracle_cfg(D, K, S, missing, F, T):
    w_cls, f_cls = L.tree_cls(D)
    return O.make_cfg(D, K, S, missing, w_cls, f_cls, F // 4, T)


def oracle_scores(W, FI, x, D, K, S, missing, **kw):
    wl, fl = L.pack_streams(W, FI, D)
    cfg = oracle_cfg(D, K, S, missing, x.shape[1], W.shape[0])
    return O.scores(cfg, wl, fl, x, **kw)


def oracle_words(W, FI, x, D, K, S, C, missing=L.MISSING_DEFAULT):
    """uint32 words [n] (C = 1) or [n, C]: column c is the oracle's score of the class-c trees alone (tree t of the
    stream belongs to class t % C); a class without trees scores +0."""
    kw = dict(threads=O.max_threads())
    if C == 1:
        return oracle_scores(W, FI, x, D, K, S, missing, **kw)
    out = np.zeros((x.shape[0], C), dtype=np.uint32)
    for c in range(C):
        if W[c::C].shape[0]:
            out[:, c] = oracle_scores(W[c::C], FI[c::C], x, D, K, S, missing, **kw)
    return out


def labels_of(words, C):
    """The labels of score words: C = 1: score > 0 (label 0 at +0); C >= 2: the first class of maximal score."""
    return O.labels(words) if C == 1 else np.argmax(words.view(np.float32), axis=1).astype(np.uint8)


def geometry_regs(T, D, F, K, S, missing, n_tuples=0):
    """Register values 201..208 for an explicit (K, S) — S may differ from the profile default."""
    regs = E.csr_from_profile(T, D, 4 * F, K, missing, n_tuples)
    r205 = regs[205]
    r205 = (r205 & ~(0xFF << 36)) | ((S & 0xFF) << 36)
    regs[205] = r205
    return regs


def multi_node_regs(T, D, F, K, n, ndev, mode, batch_tuples=2):
    """Register values of a multi-device run as a Catapult host would write them (EngineCSR.sv:194-216)."""
    w_cls, f_cls = L.tree_cls(D)
    per = -(-T // ndev)
    regs = E.csr_from_profile(T, D, 4 * F, K, L.MISSING_DEFAULT, n)
    flags = 0x2 | 0x20 | 0x40                       # host_node | multiple_nodes | pcie_receiver_enabled
    if mode == "ensemble":
        flags |= 0x4 | 0x10                         # broadcast_data | aggreg_enabled
        S = -(-per // (8 * K))
        regs[205] = (regs[205] & ~(0xFF << 36)) | (S << 36)
    else:
        flags |= 0x8                                # broadcast_trees
    regs[201] = flags | ((batch_tuples * (F // 4)) << 32)
    regs[203] = ((per * w_cls - 1) & 0xFFFF) | ((per * f_cls) << 16) | (ndev << 32)
    return regs


def write_regs(e, regs):
    for a, v in sorted(regs.items()):
        e.softreg_write(a, v)


def make_engine(T, D, F, K=8, S=None, missing=L.MISSING_DEFAULT, n_tuples=0, gpus=0):
    """An engine on `gpus` with the geometry registers of T trees of depth D on F features written; S = None: the
    fewest slots that hold T trees with K partials."""
    e = ddt.Engine(gpus)
    S = S if S is not None else max(1, -(-T // (8 * K)))
    write_regs(e, geometry_regs(T, D, F, K, S, missing, n_tuples))
    return e


def early(FI, D, seed, root_tree=2):
    """Bit 14 (an early leaf) on one random node of every tree but the first, and on the root of tree `root_tree` when
    the ensemble has it (None: on no root)."""
    rng = np.random.default_rng(seed)
    FI = FI.copy()
    for t in range(1, FI.shape[0]):
        lvl = int(rng.integers(0, D))
        FI[t, (1 << lvl) - 1 + int(rng.integers(0, 1 << lvl))] |= 1 << 14
    if root_tree is not None and FI.shape[0] > root_tree:
        FI[root_tree, 0] |= 1 << 14
    return FI


# ---- the plan tables -------------------------------------------------------------------------------------------------
class Row(collections.namedtuple("Row", "tune D F C variant name")):
    @property
    def template(self):
        """Kernel template of the row: "dt_walk_tile<4, 2, 1, 0, 384>" or "dt_walk_generic<1>"."""
        return self.name.split(">")[0] + ">"


def plan_rows(table_file):
    """Rows of tests/golden/<table_file> in file order: (DTE_TUNE pin, D, F, C, requested variant, kernel name)."""
    rows, tune = [], None
    with lzma.open(os.path.join(HERE, "golden", table_file), "rt") as f:
        for line in f:
            line = line.rstrip("\n")
            if line.startswith("DTE_TUNE="):
                tune = line[len("DTE_TUNE="):]
                continue
            D, F, C, variant, _phased, name = line.split(" ", 5)
            rows.append(Row(tune, int(D), int(F), int(C), int(variant), name))
    return rows


def plan_groups(rows):
    """{(template, C): (typical row, extreme row)}, groups in order of first appearance.  Typical: the smallest
    (|D - 10|, F), extreme: the largest (D, F); ties go to the first row in table order."""
    groups = collections.OrderedDict()
    for r in rows:
        groups.setdefault((r.template, r.C), []).append(r)
    return collections.OrderedDict((k, (min(rs, key=lambda r: (abs(r.D - 10), r.F)), max(rs, key=lambda r: (r.D, r.F))))
                                   for k, rs in groups.items())


# ---- the device ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    assert torch.cuda.is_available(), "these tests need the H100"
    return torch


def device_rows(torch, e, sfx, x, row_shape, dtype=np.float32, stream=None):
    """[n, *row_shape] of `dtype` from e.infer_device<sfx>, written to a buffer with canary words after the last row."""
    n, row = x.shape[0], int(np.prod(row_shape))
    dx = torch.from_numpy(np.ascontiguousarray(x).view(np.int32)).cuda()
    buf = torch.full((n * row + 64,), CANARY, dtype=torch.int32, device="cuda")
    getattr(e, "infer_device" + sfx)(dx, n, buf, stream=stream)
    torch.cuda.synchronize()
    got = buf.cpu().numpy()
    assert (got[n * row:] == CANARY).all(), "wrote past the last row"
    return got[: n * row].view(dtype).reshape((n,) + tuple(row_shape))


def device_scores(torch, e, sfx, x, C, stream=None):
    """Score words [n] or [n, C] and labels from e.infer_device<sfx>, with canaries after the last score and label."""
    n = x.shape[0]
    dx = torch.from_numpy(np.ascontiguousarray(x).view(np.int32)).cuda()
    buf = torch.full((n * C + 64,), CANARY, dtype=torch.int32, device="cuda")
    lb = torch.full((n + 16,), 0xA5, dtype=torch.uint8, device="cuda")
    getattr(e, "infer_device" + sfx)(dx, n, buf, lb, stream=stream)
    torch.cuda.synchronize()
    got, labels = buf.cpu().numpy(), lb.cpu().numpy()
    assert (got[n * C:] == CANARY).all(), "wrote past the last score"
    assert (labels[n:] == 0xA5).all(), "wrote past the last label"
    sc = got[: n * C].view(np.uint32)
    return (sc if C == 1 else sc.reshape(n, C)), labels[:n]


def host_rows(e, sfx, x, C):
    """e.infer_host<sfx>(x) with the class axis kept when C = 1."""
    out = getattr(e, "infer_host" + sfx)(x)
    return out[:, None] if C == 1 else out


U = 2.0 ** -24


def efficiency(torch, e, x, phi, leaf_abs, T):
    """phi [n, C, F + 1] against the same handle's dte_infer_device score words: sum_f phi + bias is the score up to one
    fp32 rounding of every word (U |word|), the fp64 roundings before them (far below 1e-12 of the leaf magnitudes
    leaf_abs) and the score word's (T + 1) fp32 roundings of its leaf sum."""
    n, C = x.shape[0], phi.shape[1]
    dx = torch.from_numpy(np.ascontiguousarray(x).view(np.int32)).cuda()
    ds = torch.empty(n * C, dtype=torch.float32, device="cuda")
    e.infer_device(dx, n, ds)
    score = ds.cpu().numpy().astype(np.float64).reshape(n, C)
    p = phi.astype(np.float64)
    bound = U * np.abs(p).sum(axis=2) + (T + 1) * U * leaf_abs + 1e-12 * leaf_abs
    assert (np.abs(p.sum(axis=2) - score) <= bound).all()


# ---- checks ----------------------------------------------------------------------------------------------------------
def _bits(a):
    a = np.asarray(a)
    return a.view(np.uint32) if a.dtype == np.float32 else a


def assert_words(got, want, what):
    """Equal word for word (fp32 compared by its bits), in the same shape; the message names the first difference."""
    g, w = _bits(got), _bits(want)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    bad = np.argwhere(g != w)
    assert bad.size == 0, "%s: %d words differ, first at %s: %#x instead of %#x" % (
        what, len(bad), tuple(bad[0]), g[tuple(bad[0])], w[tuple(bad[0])])


def assert_scores(sc, lb, want, C, what):
    """Score words sc (any shape of want's size) equal to the words want, and labels lb (None: not checked) equal to
    labels_of(want, C)."""
    assert_words(_bits(sc).reshape(want.shape), want, what)
    if lb is not None:
        lw = labels_of(want, C)
        bad = np.flatnonzero(np.asarray(lb) != lw)
        assert bad.size == 0, "%s: %d labels differ, first at tuple %d: got %d want %d" % (
            what, bad.size, bad[0], lb[bad[0]], lw[bad[0]])


def refused(call, code, *needles):
    """call() raises DteError with status `code` and a message containing every needle; returns the message."""
    with pytest.raises(E.DteError) as ex:
        call()
    msg = str(ex.value)
    assert ex.value.code == code, msg
    for s in needles:
        assert s in msg, msg
    return msg


def refused_exactly(call, code, message):
    """refused(), with the whole message pinned: "dte error <code>: <message>"."""
    assert refused(call, code) == "dte error %d: %s" % (code, message)
