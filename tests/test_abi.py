"""The C-ABI library loads on a CPU-only box and exports every symbol include/dte.h declares.
No compute call is made here (there is no GPU and no CPU fallback)."""
import ctypes as C
import os
import re

import pytest

import ddt_b200 as ddt
from ddt_b200 import engine as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_source():
    src = open(os.path.join(ROOT, "include", "dte.h")).read()
    return re.sub(r"/\*.*?\*/", "", src, flags=re.S)


def header_symbols():
    return sorted(set(re.findall(r"\b(dte_[a-z_0-9]+)\s*\(", header_source())))


def test_library_exports_every_declared_symbol():
    lib = ddt.load_library()
    syms = header_symbols()
    assert len(syms) >= 24
    for s in syms:
        assert hasattr(lib, s), "libdte.so does not export %s" % s
    # and the Python mirror binds exactly the header's set
    assert sorted(n for n, _, _ in E.ABI) == syms


def test_status_codes_match_the_header():
    """Every value of the dte_status enum in include/dte.h, and the Python mirror of it in engine.py."""
    body = re.search(r"typedef enum \{([^}]*)\} dte_status;", header_source()).group(1)
    codes = {name: int(value) for name, value in re.findall(r"\b(DTE_\w+)\s*=\s*(-?\d+)", body)}
    assert codes["DTE_OK"] == 0 and len(codes) == 8, codes
    for name, value in codes.items():
        assert getattr(E, name) == value, name


def test_version_string():
    assert b"sm_90a" in ddt.load_library().dte_version()


def test_csr_from_profile_worked_examples():
    # SURVEY.md §8b worked examples (derived from EngineCSR.sv field definitions)
    r = E.csr_from_profile(16, 4, 128, clusters=2, missing_value=0xBF800000, n_tuples=10000)
    assert (r[204] >> 16) & 0xFFFF == 8          # weights CLs / tree = ceil(31/4)
    assert (r[204] >> 32) & 0xFFFF == 2          # findex CLs / tree = ceil(15/8)
    assert (r[204] >> 48) & 0xFFFF == 8          # tuple CLs
    assert r[204] & 0xFF == 0x55 and (r[204] >> 8) & 0xFF == 0x03
    assert r[202] >> 32 == 128 and r[202] & 0xFFFFFFFF == 160
    assert (r[205] >> 32) & 0xF == 4 and (r[205] >> 36) & 0xFF == 1 and (r[205] >> 44) & 0xF == 2
    assert r[205] & 0xFFFFFFFF == 0xBF800000
    assert r[207] & 0xFFFFFFFF == 2500
    assert r[201] & 0xFF == 0x42
    r = E.csr_from_profile(1024, 12, 1024, clusters=8, n_tuples=50_000_000)
    assert (r[204] >> 16) & 0xFFFF == 2048 and (r[204] >> 32) & 0xFFFF == 512 and (r[204] >> 48) & 0xFFFF == 64
    assert r[202] >> 32 == 2_097_152 and r[202] & 0xFFFFFFFF == 2_621_440
    assert (r[205] >> 36) & 0xFF == 16 and (r[205] >> 44) & 0xF == 8
    assert r[204] & 0xFF == 0x01 and (r[204] >> 8) & 0xFF == 0xFF
    assert r[207] & 0xFFFFFFFF == 12_500_000


@pytest.mark.parametrize("args", [
    (0, 4, 128, 2), (16, 0, 128, 2), (16, 16, 128, 2), (16, 4, 100, 2), (16, 4, 128, 3), (16, 4, 0, 1),
    (100000, 4, 128, 1),    # S would not fit the 8-bit field
])
def test_csr_from_profile_rejects_bad_parameters(args):
    with pytest.raises(E.DteError):
        E.csr_from_profile(args[0], args[1], args[2], clusters=args[3])


def test_no_cpu_fallback_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(E.DteError) as ei:
        ddt.Engine(0)
    assert ei.value.code == E.DTE_ERR_CUDA


def test_null_arguments_are_errors_not_crashes():
    lib = ddt.load_library()
    assert lib.dte_create(None, 0) == E.DTE_ERR_ARG
    assert lib.dte_destroy(None) == E.DTE_ERR_ARG
    assert lib.dte_softreg_write(None, 200, 1) == E.DTE_ERR_ARG
    v = C.c_uint64()
    assert lib.dte_softreg_read(None, 220, C.byref(v)) == E.DTE_ERR_ARG
    assert lib.dte_last_error(None) == b"null engine"
    assert lib.dte_set_node(None, 0) == E.DTE_ERR_ARG


def test_product_does_not_touch_the_oracle():
    # the product path must never import, link or call anything under oracle/
    pkg = os.path.join(ROOT, "distributed-decisiontrees_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "dteo_" not in txt and "libdte_oracle" not in txt and "from oracle" not in txt, f
    import subprocess
    out = subprocess.run(["nm", "-D", ddt.lib_path()], capture_output=True, text=True).stdout
    assert "dteo_" not in out
