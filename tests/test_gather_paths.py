"""tools/gather_paths.py walks the top levels with the oracle's rule: the record it reports, walked two more levels,
reaches the leaf dteo_leaf returns (missing features included)."""
import ctypes as C
import importlib.util
import os

import numpy as np

import ddt_b200 as ddt
from oracle import oracle as O

L = ddt.layout
_TOOL = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "gather_paths.py")
_spec = importlib.util.spec_from_file_location("gather_paths", _TOOL)
GP = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(GP)


def s32(u):
    return u - (1 << 32) if u >= 1 << 31 else u


def test_records_lead_to_the_oracle_leaf():
    T, D, F, n = 6, 7, 48, 96
    W, FI = L.synth_ensemble(T, D, F)
    x = L.synth_tuples(0, n, F, missing_ppm=150_000)
    assert (x == L.MISSING_DEFAULT).any()
    J = GP.records(W, FI.astype(np.int64), D, x.view(np.int32))
    assert J.shape == (T, n) and int(J.max()) < 1 << (D - 2)
    w_cls, f_cls = L.tree_cls(D)
    cfg = O.make_cfg(D, 8, 1, L.MISSING_DEFAULT, w_cls, f_cls, F // 4, T)
    lib = O.lib()
    for t in range(T):
        w = np.ascontiguousarray(W[t], dtype=np.uint32)
        fi = np.ascontiguousarray(FI[t], dtype=np.uint16)
        for m in range(n):
            row = np.ascontiguousarray(x[m])
            nd = (1 << (D - 2)) - 1 + int(J[t, m])
            for _ in range(2):
                f = int(fi[nd])
                v = int(row[f & 0x7FF])
                right = (f >> 13) & 1 if v == L.MISSING_DEFAULT else int(not (s32(v) < s32(int(w[nd]))))
                nd = 2 * nd + 1 + right
            want = lib.dteo_leaf(C.byref(cfg), w.ctypes.data, fi.ctypes.data, row.ctypes.data)
            assert int(w[nd]) == want, (t, m)
