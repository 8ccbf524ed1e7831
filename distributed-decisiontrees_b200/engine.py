"""ctypes mirror of include/dte.h — the host-side view of the engine.

Method names follow the reference's own interface vocabulary (soft registers, 128-bit line
streams; rtl/DTEngine/EngineCSR.sv, rtl/DTEngine/PCIeReceiver.sv) so the parity tests read like a
Catapult host program.  There is no Python compute path here: every score comes out of libdte.so's
CUDA kernels, and loading fails loudly when the library is missing.
"""
import ctypes as C
import os

import numpy as np

from . import build as _build

_HERE = os.path.dirname(os.path.abspath(__file__))

DTE_KERNEL_AUTO, DTE_KERNEL_GENERIC, DTE_KERNEL_TILE, DTE_KERNEL_TILE_STAGED = 0, 1, 2, 3
KERNEL_NAMES = {0: "auto", 1: "generic", 2: "tile", 3: "tile_staged"}

# every symbol include/dte.h declares: (name, restype, argtypes)
_u64p = C.POINTER(C.c_uint64)
ABI = [
    ("dte_create", C.c_int, [C.POINTER(C.c_void_p), C.c_int]),
    ("dte_create_multi", C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.c_int]),
    ("dte_set_option", C.c_int, [C.c_void_p, C.c_int, C.c_uint64]),
    ("dte_stream_flush", C.c_int, [C.c_void_p]),
    ("dte_ring_combine_device", C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("dte_destroy", C.c_int, [C.c_void_p]),
    ("dte_last_error", C.c_char_p, [C.c_void_p]),
    ("dte_softreg_write", C.c_int, [C.c_void_p, C.c_uint32, C.c_uint64]),
    ("dte_softreg_read", C.c_int, [C.c_void_p, C.c_uint32, _u64p]),
    ("dte_stream_write", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    ("dte_stream_read", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("dte_stream_read_packets", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("dte_process_done", C.c_int, [C.c_void_p, C.POINTER(C.c_int)]),
    ("dte_load_ensemble", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32]),
    ("dte_load_ensemble_classes", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32,
                                            C.c_uint32]),
    ("dte_infer_device", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("dte_infer_host", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("dte_infer_device_accumulate", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("dte_ipc_alloc", C.c_int, [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p), C.c_char_p]),
    ("dte_ipc_open", C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p)]),
    ("dte_ipc_close", C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    ("dte_host_alloc", C.c_int, [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p)]),
    ("dte_host_free", C.c_int, [C.c_void_p, C.c_void_p]),
    ("dte_labels_device", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("dte_class_labels_device", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_void_p]),
    ("dte_ring_add_device", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    ("dte_csr_from_profile", C.c_int, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint64, _u64p]),
    ("dte_get_info", C.c_int, [C.c_void_p, C.c_void_p]),
    ("dte_set_kernel_variant", C.c_int, [C.c_void_p, C.c_int]),
    ("dte_kernel_name", C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t]),
    ("dte_autotune", C.c_int, [C.c_void_p, C.c_size_t, C.c_char_p, C.c_size_t]),
    ("dte_set_node", C.c_int, [C.c_void_p, C.c_uint32]),
    ("dte_synth_tuples_device", C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint64,
                                           C.c_uint32, C.c_uint32, C.c_void_p]),
    ("dte_version", C.c_char_p, []),
    ("dte_load_ensemble_binned", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32,
                                           C.c_uint32]),
    ("dte_bin_edges", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]),
    ("dte_bin_tuples_device", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("dte_infer_device_binned", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("dte_infer_host_binned", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("dte_kernel_name_binned", C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t]),
    ("dte_infer_device_leaves", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("dte_infer_host_leaves", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    ("dte_kernel_name_leaves", C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t]),
    ("dte_load_ensemble_contribs", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint32,
                                             C.c_uint32, C.c_uint32]),
    ("dte_infer_device_contribs", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("dte_infer_host_contribs", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    ("dte_kernel_name_contribs", C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t]),
    ("dte_infer_device_interactions", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("dte_infer_host_interactions", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    ("dte_kernel_name_interactions", C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t]),
    ("dte_load_ensemble_approx_contribs", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                                    C.c_uint32, C.c_uint32, C.c_uint32]),
    ("dte_infer_device_approx_contribs", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("dte_infer_host_approx_contribs", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    ("dte_kernel_name_approx_contribs", C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t]),
    ("dte_load_ensemble_interventional", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_uint32,
                                                   C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t]),
    ("dte_infer_device_interventional", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("dte_infer_host_interventional", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    ("dte_kernel_name_interventional", C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t]),
    ("dte_load_ensemble_categorical", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_uint32,
                                                C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p]),
    ("dte_infer_device_categorical", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]),
    ("dte_infer_host_categorical", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]),
    ("dte_kernel_name_categorical", C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t]),
    ("dte_sparse_to_dense_device", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64,
                                             C.c_void_p, C.c_void_p]),
    ("dte_infer_device_sparse", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p,
                                          C.c_void_p, C.c_void_p]),
    ("dte_infer_host_sparse", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p,
                                        C.c_void_p]),
]


class DteInfo(C.Structure):
    _fields_ = [
        ("num_trees", C.c_uint32), ("num_levels", C.c_uint32), ("num_features", C.c_uint32),
        ("clusters", C.c_uint32), ("trees_per_pu", C.c_uint32), ("kernel_variant", C.c_uint32),
        ("tuples_per_cta", C.c_uint32), ("sm_count", C.c_uint32), ("ensemble_bytes", C.c_uint64),
        ("kernel_launches", C.c_uint64), ("last_walk_ms", C.c_double),
        ("num_devices", C.c_uint32), ("partition", C.c_uint32), ("tuples_in", C.c_uint64), ("tuples_out", C.c_uint64),
        ("num_classes", C.c_uint32), ("plan_source", C.c_uint32),
    ]


PLAN_SOURCES = {0: "static", 1: "measured"}    # dte_plan_source


DTE_OPT_CYCLE_MHZ, DTE_OPT_COMBINE, DTE_OPT_RESULT_QUEUE_LINES, DTE_OPT_CHUNK_TUPLES = 1, 2, 3, 4
DTE_OPT_LEAF_LAYOUT = 5
DTE_OPT_INTERACTION_BLOCK = 6     # matrix rows per interaction pass (0 = the planner's)
DTE_OK = 0
DTE_ERR_ARG, DTE_ERR_STATE, DTE_ERR_CONFIG, DTE_ERR_UNSUPPORTED, DTE_ERR_CUDA, DTE_ERR_NOMEM = -1, -2, -3, -4, -5, -6
DTE_ERR_BACKPRESSURE = -7
DTE_SPARSE_ABSENT_MISSING = 0xFFFFFFFFFFFFFFFF   # sparse calls: an absent feature is the run's missing pattern (reg 205)
CUDA_STREAM_LEGACY = 0x1        # cudaStreamLegacy: the handle value that NAMES the legacy default stream


class DteError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("dte error %d: %s" % (code, msg))
        self.code = code


def lib_path():
    return os.path.join(_HERE, "libdte.so")


def build_library(force=False, verbose=False):
    return _build.build(force=force, verbose=verbose)


_LIB = None


def load_library(rebuild_if_stale=True):
    """dlopen the in-tree libdte.so (building it with nvcc when sources are newer) and bind the ABI."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if rebuild_if_stale and _build.nvcc_path() is not None and _build.stale():
        _build.build()
    if not os.path.exists(path):
        raise RuntimeError("libdte.so is missing and cannot be built here — the engine has no CPU fallback")
    lib = C.CDLL(path)
    for name, res, args in ABI:
        fn = getattr(lib, name)          # AttributeError if the header and the library disagree
        fn.restype = res
        fn.argtypes = args
    _LIB = lib
    return lib


def csr_from_profile(n_trees, depth_levels, tuple_bytes, clusters=8, missing_value=0xBF800000, n_tuples=0):
    """profiler.cpp's three inputs (N_trees, Depth_tree, Size_tuple_Bytes) -> {register: value}."""
    lib = load_library()
    regs = (C.c_uint64 * 8)()
    rc = lib.dte_csr_from_profile(n_trees, depth_levels, tuple_bytes, clusters, missing_value, n_tuples, regs)
    if rc:
        raise DteError(rc, "dte_csr_from_profile rejected the parameters")
    return {201 + i: int(regs[i]) for i in range(8)}


def _stream(stream):
    """cudaStream_t for the C ABI.  None -> NULL (the engine's own stream, synchronous call).  An int is a raw
    cudaStream_t; torch reports the legacy default stream as 0, which the ABI reads as NULL, so 0 is translated to
    cudaStreamLegacy (0x1) — the call then really runs on, and is ordered with, the caller's default stream."""
    if stream is None:
        return None
    s = int(stream)
    return C.c_void_p(s if s else CUDA_STREAM_LEGACY)


def _ptr(x):
    """Device/host address of a numpy array, a torch tensor, an int, or None."""
    if x is None:
        return None
    if isinstance(x, int):
        return C.c_void_p(x)
    if isinstance(x, np.ndarray):
        return C.c_void_p(x.ctypes.data)
    if hasattr(x, "data_ptr"):
        return C.c_void_p(x.data_ptr())
    raise TypeError("cannot take the address of %r" % type(x))


def _absent(absent):
    """The `absent` argument of the sparse calls: None -> DTE_SPARSE_ABSENT_MISSING, else the word as given."""
    return DTE_SPARSE_ABSENT_MISSING if absent is None else int(absent)


def _host_rows(x, dtype=None):
    """(rows, n) of a host array [n, ...]: a numpy array made C-contiguous (and of `dtype` when given), or a pinned torch
    CPU tensor as it is."""
    if isinstance(x, np.ndarray):
        x = np.ascontiguousarray(x, dtype=dtype)
    return x, int(x.shape[0])


class Engine:
    """One in-order engine on one GPU (the analogue of one FPGA role)."""

    def __init__(self, gpu_ordinal=0):
        """gpu_ordinal: one CUDA ordinal, or a list of ordinals = one handle driving the whole ring of devices
        (dte_create_multi; ordinals[d] is device ID d of `devices_list`)."""
        self._lib = load_library()
        self._h = C.c_void_p()
        if isinstance(gpu_ordinal, (list, tuple)):
            arr = (C.c_int * len(gpu_ordinal))(*[int(g) for g in gpu_ordinal])
            rc = self._lib.dte_create_multi(C.byref(self._h), arr, len(gpu_ordinal))
            self.gpu = int(gpu_ordinal[0]) if gpu_ordinal else 0
            self.gpus = [int(g) for g in gpu_ordinal]
        else:
            rc = self._lib.dte_create(C.byref(self._h), int(gpu_ordinal))
            self.gpu = int(gpu_ordinal)
            self.gpus = [self.gpu]
        if rc:
            self._h = C.c_void_p()
            raise DteError(rc, "dte_create failed (no CUDA device? there is no CPU fallback)")

    # -- plumbing ---------------------------------------------------------------------------
    def _check(self, rc):
        if rc:
            raise DteError(rc, self._lib.dte_last_error(self._h).decode())

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self._lib.dte_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # -- soft registers (EngineCSR.sv) --------------------------------------------------------
    def softreg_write(self, addr, data):
        if int(addr) == 200 and int(data) & 1:
            self._classes = None                         # `start`: a tree stream may place a new ensemble
        self._check(self._lib.dte_softreg_write(self._h, int(addr), int(data) & 0xFFFFFFFFFFFFFFFF))
        self._written = getattr(self, "_written", {})
        self._written[int(addr)] = int(data) & 0xFFFFFFFFFFFFFFFF    # reads return status counters, not these words

    def softreg_read(self, addr):
        v = C.c_uint64()
        self._check(self._lib.dte_softreg_read(self._h, int(addr), C.byref(v)))
        return int(v.value)

    def configure(self, n_trees, depth_levels, tuple_bytes, clusters=8, missing_value=0xBF800000, n_tuples=0,
                  overrides=None):
        """Write registers 201..208 derived from the profiler-style parameters; returns them."""
        regs = csr_from_profile(n_trees, depth_levels, tuple_bytes, clusters, missing_value, n_tuples)
        if overrides:
            regs.update(overrides)
        for a, v in sorted(regs.items()):
            self.softreg_write(a, v)
        return regs

    def start(self):
        self.softreg_write(200, 1)

    # -- 128-bit line streams (PCIeReceiver.sv / ResultsCombiner.sv) -----------------------------
    def stream_write(self, lines):
        a = np.ascontiguousarray(lines)
        nbytes = a.nbytes
        if nbytes % 16:
            raise ValueError("stream_write needs whole 128-bit lines")
        self._check(self._lib.dte_stream_write(self._h, _ptr(a), nbytes // 16))

    def stream_read(self, max_lines):
        out = np.empty((int(max_lines), 4), dtype=np.float32)
        got = C.c_size_t()
        self._check(self._lib.dte_stream_read(self._h, _ptr(out), int(max_lines), C.byref(got)))
        return out[: got.value]

    def stream_read_packets(self, max_lines):
        """-> (result lines [n, 4] fp32, last flags [n] u8): `last` closes a PCIe packet (DTInference.sv:659-663)."""
        out = np.empty((int(max_lines), 4), dtype=np.float32)
        last = np.zeros(int(max_lines), dtype=np.uint8)
        got = C.c_size_t()
        self._check(self._lib.dte_stream_read_packets(self._h, _ptr(out), _ptr(last), int(max_lines), C.byref(got)))
        return out[: got.value], last[: got.value]

    def stream_flush(self):
        self._check(self._lib.dte_stream_flush(self._h))

    def set_option(self, option, value):
        self._check(self._lib.dte_set_option(self._h, int(option), int(value)))
        if int(option) == DTE_OPT_LEAF_LAYOUT:
            self._leaf_opt = int(value)

    def ring_combine_device(self, d_parts, n, d_out, d_labels=None, stream=None):
        """out = (((p0 + p1) + p2) + ...) in ring order, one kernel; d_parts may be peer-GPU buffers."""
        arr = (C.c_void_p * len(d_parts))(*[_ptr(p) for p in d_parts])
        self._check(self._lib.dte_ring_combine_device(self._h, arr, len(d_parts), int(n), _ptr(d_out), _ptr(d_labels),
                                                      _stream(stream)))

    def stream_read_into(self, out_lines, last_flags=None, offset=0):
        """Zero-copy variant: result lines go straight into out_lines[offset:] ([n, 4] fp32, C-contiguous) and the packet
        flags into last_flags[offset:] (u8); returns the number of lines read."""
        room = out_lines.shape[0] - int(offset)
        got = C.c_size_t()
        po = C.c_void_p(out_lines.ctypes.data + 16 * int(offset))
        pl = C.c_void_p(last_flags.ctypes.data + int(offset)) if last_flags is not None else None
        self._check(self._lib.dte_stream_read_packets(self._h, po, pl, room, C.byref(got)))
        return int(got.value)

    def process_done(self):
        d = C.c_int()
        self._check(self._lib.dte_process_done(self._h, C.byref(d)))
        return bool(d.value)

    # -- fast paths -----------------------------------------------------------------------------
    def load_ensemble(self, weight_cls, findex_cls, first_tree=0, num_local_trees=0, num_classes=1, binned=False,
                      leaves=False, covers=None, approx=False, background=None, categories=None):
        """num_classes >= 2: a multi-class ensemble, tree t of the stream belongs to class t % num_classes; every infer
        call then returns [n, num_classes] scores and argmax labels (dte_load_ensemble_classes).
        binned=True: also build the binned layout (dte_load_ensemble_binned; at most 254 distinct live thresholds per
        feature), which the *_binned calls walk with u8 tuples.
        leaves=True: DTE_OPT_LEAF_LAYOUT = 1 for this load, so the *_leaves calls can walk it.
        covers: fp32 [T_all, 2^(D+1)-1] node covers of every tree of the streams, indexed like the weight heap: also build
        the contribution layout the *_contribs calls walk (dte_load_ensemble_contribs; not with binned=True).
        approx=True (with covers): build the approximate-contribution table and the leaf-id layout instead, which the
        *_approx_contribs and *_leaves calls walk (dte_load_ensemble_approx_contribs; not with binned=True).
        background: [N, F] float32 (or uint32 words) background rows: build the interventional layout the *_interventional
        calls walk (dte_load_ensemble_interventional; not with covers, approx=True or binned=True).
        categories: (set_offsets uint32 [n_sets + 1], set_words uint32) CSR category sets: a live node with bit 15 of its
        feature-index word tests x[f]'s category against set W[n] (dte_load_ensemble_categorical); the *_categorical calls
        walk it and every other call is refused until the next load.  Not with binned=True, covers, approx=True or
        background; (None, None) or empty arrays: no sets."""
        w = np.ascontiguousarray(weight_cls)
        f = np.ascontiguousarray(findex_cls)
        self._classes = None
        if background is not None and (covers is not None or approx or binned):
            raise ValueError("background cannot be combined with covers, approx=True or binned=True: one attribution layout "
                             "is resident at a time, and the interventional calls take fp32 tuples")
        if categories is not None and (binned or covers is not None or approx or background is not None):
            raise ValueError("categories cannot be combined with binned=True, covers, approx=True or background: a "
                             "categorical layout is resident alone and only the categorical calls walk it")
        if approx and binned:
            raise ValueError("approx and binned=True cannot be combined: the approximate contribution calls take fp32 tuples")
        if approx and covers is None:
            raise ValueError("approx=True needs covers: the table is built from the node covers")
        args = (_ptr(w), w.nbytes // 16, _ptr(f), f.nbytes // 16)
        tail = (int(first_tree), int(num_local_trees), int(num_classes))
        if categories is not None:
            offs, words = categories
            offs = np.ascontiguousarray(offs if offs is not None else np.zeros(0), dtype=np.uint32)
            words = np.ascontiguousarray(words if words is not None and np.size(words) else np.zeros(1), dtype=np.uint32)
            n_sets = max(0, offs.size - 1)
            self._cat_sets = (offs, words)           # kept alive for the call
            kind, args = "categorical", args + tail + ((_ptr(offs), n_sets, _ptr(words)) if n_sets else (None, 0, None))
        elif background is not None:
            bg = np.asarray(background)
            r204 = getattr(self, "_written", {}).get(204)
            F = ((r204 >> 48) & 0xFFFF) * 4 if r204 is not None else None   # tuple lines of register 204, four words each
            if bg.dtype not in (np.float32, np.uint32) or bg.ndim != 2 or F is None or bg.shape[1] != F:
                raise ValueError("background must be a [N, F] float32 or uint32 array with F from register 204 (%s), "
                                 "not %s %s" % (F if F is not None else "not written", bg.dtype, bg.shape))
            bg = np.ascontiguousarray(bg).view(np.uint32)
            kind, args = "interventional", args + tail + (_ptr(bg), int(bg.shape[0]))
        elif covers is not None:
            if binned:
                raise ValueError("covers and binned=True cannot be combined: the contribution calls take fp32 tuples")
            cv = np.ascontiguousarray(covers, dtype=np.float32)
            kind, args = "approx_contribs" if approx else "contribs", args + (_ptr(cv),) + tail
        else:
            kind, args = "binned" if binned else "classes", args + tail
        saved = getattr(self, "_leaf_opt", 0)
        if leaves:
            self.set_option(DTE_OPT_LEAF_LAYOUT, 1)
        try:
            self._check(getattr(self._lib, "dte_load_ensemble_" + kind)(self._h, *args))
        finally:
            if leaves:
                self.set_option(DTE_OPT_LEAF_LAYOUT, saved)
        self._classes = int(num_classes)

    def num_classes(self):
        """Score words per tuple of the resident ensemble (1 for a single-class ensemble)."""
        c = getattr(self, "_classes", None)
        if c is None:                                    # e.g. placed by a tree line stream: ask the engine
            c = max(1, int(self.info()["num_classes"]))
            self._classes = c
        return c

    def infer_device(self, d_tuples, n, d_scores, d_labels=None, stream=None):
        """d_* are device pointers (ints) or torch CUDA tensors; stream is a cudaStream_t int (None = engine stream, synchronous)."""
        self._check(self._lib.dte_infer_device(self._h, _ptr(d_tuples), int(n), _ptr(d_scores), _ptr(d_labels),
                                               _stream(stream)))

    def _score_outputs(self, n, want_labels, out_scores, out_labels):
        """The (scores, labels) a host-buffer score call of n tuples writes: the caller's arrays, else new ones."""
        if out_scores is None:
            nc = self.num_classes()
            out_scores = np.empty(n, dtype=np.float32) if nc == 1 else np.empty((n, nc), dtype=np.float32)
        if out_labels is None and want_labels:
            out_labels = np.empty(n, dtype=np.uint8)
        return out_scores, out_labels

    def _infer_host(self, fn, rows, dtype, want_labels, out_scores, out_labels):
        """Allocate the outputs of a host-buffer score call and run it -> (scores, labels)."""
        t, n = _host_rows(rows, dtype)
        scores, labels = self._score_outputs(n, want_labels, out_scores, out_labels)
        self._check(fn(self._h, _ptr(t), n, _ptr(scores), _ptr(labels)))
        return scores, labels

    def _infer_host_rows(self, fn, tuples, out, row_shape, dtype=np.float32):
        """Run a host-buffer row call of fp32 tuples [n, F] into out, else into a new array [n, *row_shape()] -> out."""
        t, n = _host_rows(tuples)
        if out is None:
            out = np.empty((n,) + row_shape(), dtype=dtype)
        self._check(fn(self._h, _ptr(t), n, _ptr(out)))
        return out

    def _attribution_row(self, axes):
        """The row shape of an attribution call: `axes` axes of F + 1, after a class axis for a multi-class ensemble."""
        F1, nc = int(self.info()["num_features"]) + 1, self.num_classes()
        return (F1,) * axes if nc == 1 else (nc,) + (F1,) * axes

    def _name(self, fn):
        buf = C.create_string_buffer(256)
        self._check(fn(self._h, buf, 256))
        return buf.value.decode()

    def infer_host(self, tuples, want_labels=True, out_scores=None, out_labels=None):
        """tuples: host array (numpy, or a pinned torch CPU tensor) [n, F] fp32 -> (scores, labels).
        scores is [n] for a single-class ensemble and [n, C] for a C-class one (out_scores must hold n*C words)."""
        return self._infer_host(self._lib.dte_infer_host, tuples, None, want_labels, out_scores, out_labels)

    # -- binned inference (DESIGN.md §9) -----------------------------------------------------------
    def bin_edges(self):
        """-> (offsets uint32 [F + 1], edges uint32 [total]) of the resident binned layout: feature f's edges are
        edges[offsets[f]:offsets[f + 1]], sorted as int32 (layout.bin_tuples takes them as they are)."""
        F = int(self.info()["num_features"])
        offsets = np.empty(F + 1, dtype=np.uint32)
        total = C.c_size_t()
        self._check(self._lib.dte_bin_edges(self._h, _ptr(offsets), None, 0, C.byref(total)))
        edges = np.empty(max(1, total.value), dtype=np.uint32)
        self._check(self._lib.dte_bin_edges(self._h, _ptr(offsets), _ptr(edges), edges.size, C.byref(total)))
        return offsets, edges[: total.value]

    def bin_tuples_device(self, d_tuples, n, d_bins, stream=None):
        """fp32 tuples [n, F] -> u8 bins [n, F], both on the device (16-byte aligned)."""
        self._check(self._lib.dte_bin_tuples_device(self._h, _ptr(d_tuples), int(n), _ptr(d_bins), _stream(stream)))

    def infer_device_binned(self, d_bins, n, d_scores, d_labels=None, stream=None):
        """infer_device on u8 bins [n, F] in device memory."""
        self._check(self._lib.dte_infer_device_binned(self._h, _ptr(d_bins), int(n), _ptr(d_scores), _ptr(d_labels),
                                                      _stream(stream)))

    def infer_host_binned(self, bins, want_labels=True, out_scores=None, out_labels=None):
        """infer_host on u8 bins [n, F] in host memory (numpy, or a pinned torch CPU tensor) -> (scores, labels)."""
        return self._infer_host(self._lib.dte_infer_host_binned, bins, np.uint8, want_labels, out_scores, out_labels)

    def kernel_name_binned(self):
        return self._name(self._lib.dte_kernel_name_binned)

    # -- leaf-index inference (DESIGN.md §10) ----------------------------------------------------------
    def infer_device_leaves(self, d_tuples, n, d_leaves, stream=None):
        """[n, T] uint16 leaf cells of fp32 tuples [n, F] into d_leaves (both on the device, 16-byte aligned)."""
        self._check(self._lib.dte_infer_device_leaves(self._h, _ptr(d_tuples), int(n), _ptr(d_leaves), _stream(stream)))

    def infer_host_leaves(self, tuples, out=None):
        """tuples: host array [n, F] fp32 (numpy, or a pinned torch CPU tensor) -> [n, T] uint16: the cell, in tree t's
        own weight heap, of the leaf that local tree t sends each tuple to (T = info()["num_trees"])."""
        return self._infer_host_rows(self._lib.dte_infer_host_leaves, tuples, out, lambda: (int(self.info()["num_trees"]),),
                                     np.uint16)

    def kernel_name_leaves(self):
        return self._name(self._lib.dte_kernel_name_leaves)

    # -- feature contributions (DESIGN.md §12) ---------------------------------------------------------
    def infer_device_contribs(self, d_tuples, n, d_contribs, stream=None):
        """[n, C, F + 1] fp32 TreeSHAP contributions (bias last) of fp32 tuples [n, F], both on the device (d_tuples 16-byte,
        d_contribs 4-byte aligned)."""
        self._check(self._lib.dte_infer_device_contribs(self._h, _ptr(d_tuples), int(n), _ptr(d_contribs), _stream(stream)))

    def infer_host_contribs(self, tuples, out=None):
        """tuples: host array [n, F] fp32 (numpy, or a pinned torch CPU tensor) -> contributions [n, F + 1] for a
        single-class ensemble, [n, C, F + 1] for a C-class one: feature f's share of the class score, the bias last."""
        return self._infer_host_rows(self._lib.dte_infer_host_contribs, tuples, out, lambda: self._attribution_row(1))

    def kernel_name_contribs(self):
        return self._name(self._lib.dte_kernel_name_contribs)

    # -- approximate feature contributions (DESIGN.md §14) ---------------------------------------------
    def infer_device_approx_contribs(self, d_tuples, n, d_contribs, stream=None):
        """[n, C, F + 1] fp32 approximate (Saabas) contributions (bias last) of fp32 tuples [n, F], both on the device
        (d_tuples 16-byte, d_contribs 4-byte aligned)."""
        self._check(self._lib.dte_infer_device_approx_contribs(self._h, _ptr(d_tuples), int(n), _ptr(d_contribs),
                                                               _stream(stream)))

    def infer_host_approx_contribs(self, tuples, out=None):
        """tuples: host array [n, F] fp32 (numpy, or a pinned torch CPU tensor) -> approximate contributions [n, F + 1] for
        a single-class ensemble, [n, C, F + 1] for a C-class one: the change in expected score each feature's splits
        make along the tuple's path, the bias (the trees' expected score) last."""
        return self._infer_host_rows(self._lib.dte_infer_host_approx_contribs, tuples, out, lambda: self._attribution_row(1))

    def kernel_name_approx_contribs(self):
        return self._name(self._lib.dte_kernel_name_approx_contribs)

    # -- interventional contributions (DESIGN.md §15) ------------------------------------------------
    def infer_device_interventional(self, d_tuples, n, d_contribs, stream=None):
        """[n, C, F + 1] fp32 interventional SHAP values (bias last) of fp32 tuples [n, F] against the background rows of the
        load, both on the device (d_tuples 16-byte, d_contribs 4-byte aligned)."""
        self._check(self._lib.dte_infer_device_interventional(self._h, _ptr(d_tuples), int(n), _ptr(d_contribs),
                                                              _stream(stream)))

    def infer_host_interventional(self, tuples, out=None):
        """tuples: host array [n, F] fp32 (numpy, or a pinned torch CPU tensor) -> interventional contributions [n, F + 1]
        for a single-class ensemble, [n, C, F + 1] for a C-class one: feature f's share of the score's distance from the
        background mean, the bias (the mean score over the background rows) last."""
        return self._infer_host_rows(self._lib.dte_infer_host_interventional, tuples, out, lambda: self._attribution_row(1))

    def kernel_name_interventional(self):
        return self._name(self._lib.dte_kernel_name_interventional)

    # -- categorical splits (DESIGN.md §16) ----------------------------------------------------------
    def infer_device_categorical(self, d_tuples, n, d_scores, d_labels=None, stream=None):
        """infer_device against a categorical load: fp32 tuples [n, F] -> scores [n] ([n, C]) and labels, on the device."""
        self._check(self._lib.dte_infer_device_categorical(self._h, _ptr(d_tuples), int(n), _ptr(d_scores), _ptr(d_labels),
                                                           _stream(stream)))

    def infer_host_categorical(self, tuples, want_labels=True, out_scores=None, out_labels=None):
        """infer_host against a categorical load: host fp32 tuples [n, F] (category codes as fp32 values) -> (scores, labels)."""
        return self._infer_host(self._lib.dte_infer_host_categorical, tuples, None, want_labels, out_scores, out_labels)

    def kernel_name_categorical(self):
        return self._name(self._lib.dte_kernel_name_categorical)

    # -- interaction values (DESIGN.md §13) ------------------------------------------------------------
    def infer_device_interactions(self, d_tuples, n, d_inter, stream=None):
        """[n, C, F + 1, F + 1] fp32 SHAP interaction values (bias at [F, F]) of fp32 tuples [n, F], both on the device
        (d_tuples 16-byte, d_inter 4-byte aligned)."""
        self._check(self._lib.dte_infer_device_interactions(self._h, _ptr(d_tuples), int(n), _ptr(d_inter), _stream(stream)))

    def infer_host_interactions(self, tuples, out=None):
        """tuples: host array [n, F] fp32 (numpy, or a pinned torch CPU tensor) -> interaction values [n, F + 1, F + 1] for
        a single-class ensemble, [n, C, F + 1, F + 1] for a C-class one: row f sums to feature f's contribution, [F, F] is
        the bias."""
        return self._infer_host_rows(self._lib.dte_infer_host_interactions, tuples, out, lambda: self._attribution_row(2))

    def kernel_name_interactions(self):
        return self._name(self._lib.dte_kernel_name_interactions)

    # -- sparse tuples (DESIGN.md §11) ------------------------------------------------------------------
    # absent=None: an absent feature is the run's missing pattern (XGBoost); a 32-bit word, e.g. 0, is used as it is.
    def infer_host_sparse(self, X, absent=None, want_labels=True, out_scores=None, out_labels=None):
        """X: CSR rows in host memory, anything with .indptr / .indices / .data (scipy csr_matrix, csr_array) or an
        (indptr, indices, values) tuple, converted by layout.sparse_arrays -> (scores, labels) as infer_host returns them
        for the densified rows."""
        from . import layout
        indptr, indices, values = layout.sparse_arrays(X)
        n = int(indptr.shape[0]) - 1
        scores, labels = self._score_outputs(n, want_labels, out_scores, out_labels)
        self._check(self._lib.dte_infer_host_sparse(self._h, _ptr(indptr), _ptr(indices), _ptr(values), n, _absent(absent),
                                                    _ptr(scores), _ptr(labels)))
        return scores, labels

    def infer_device_sparse(self, d_indptr, d_indices, d_values, n, d_scores, d_labels=None, absent=None, stream=None):
        """infer_device on CSR rows in device memory (torch CUDA tensors or pointers: int64 indptr [n + 1], uint32 / int32
        indices, 32-bit values)."""
        self._check(self._lib.dte_infer_device_sparse(self._h, _ptr(d_indptr), _ptr(d_indices), _ptr(d_values), int(n),
                                                      _absent(absent), _ptr(d_scores), _ptr(d_labels), _stream(stream)))

    def sparse_to_dense_device(self, d_indptr, d_indices, d_values, n, d_tuples, absent=None, stream=None):
        """The densified rows [n, F] of CSR rows in device memory into d_tuples (16-byte aligned)."""
        self._check(self._lib.dte_sparse_to_dense_device(self._h, _ptr(d_indptr), _ptr(d_indices), _ptr(d_values), int(n),
                                                         _absent(absent), _ptr(d_tuples), _stream(stream)))

    def infer_device_accumulate(self, d_tuples, n, d_scores_accum, stream=None):
        """Walk and ADD the partial scores into d_scores_accum (local or peer-GPU buffer), fused in the kernel."""
        self._check(self._lib.dte_infer_device_accumulate(self._h, _ptr(d_tuples), int(n), _ptr(d_scores_accum),
                                                          _stream(stream)))

    def ipc_alloc(self, nbytes):
        """-> (device pointer, 64-byte handle) of a buffer other processes can open."""
        ptr = C.c_void_p()
        buf = C.create_string_buffer(64)
        self._check(self._lib.dte_ipc_alloc(self._h, int(nbytes), C.byref(ptr), buf))
        return int(ptr.value), bytes(buf.raw)

    def ipc_open(self, handle):
        ptr = C.c_void_p()
        self._check(self._lib.dte_ipc_open(self._h, C.c_char_p(bytes(handle)), C.byref(ptr)))
        return int(ptr.value)

    def ipc_close(self, ptr, owner):
        self._check(self._lib.dte_ipc_close(self._h, C.c_void_p(int(ptr)), 1 if owner else 0))

    def host_alloc(self, shape, dtype):
        """numpy array over page-locked, portable host memory (dte_host_alloc); release with host_free(array)."""
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        ptr = C.c_void_p()
        self._check(self._lib.dte_host_alloc(self._h, n, C.byref(ptr)))
        buf = (C.c_char * n).from_address(ptr.value)
        a = np.frombuffer(buf, dtype=dtype).reshape(shape)
        self._host_ptrs = getattr(self, "_host_ptrs", {})
        self._host_ptrs[a.ctypes.data] = ptr.value
        return a

    def host_free(self, array):
        ptr = getattr(self, "_host_ptrs", {}).pop(array.ctypes.data, None)
        if ptr is not None:
            self._check(self._lib.dte_host_free(self._h, C.c_void_p(ptr)))

    def labels_device(self, d_scores, n, d_labels, stream=None):
        self._check(self._lib.dte_labels_device(self._h, _ptr(d_scores), int(n), _ptr(d_labels),
                                                _stream(stream)))

    def class_labels_device(self, d_scores, n, num_classes, d_labels, stream=None):
        """labels[i] = first argmax over the [n, num_classes] scores (lowest class wins a tie); 1 class: score > 0."""
        self._check(self._lib.dte_class_labels_device(self._h, _ptr(d_scores), int(n), int(num_classes), _ptr(d_labels),
                                                      _stream(stream)))

    def ring_add_device(self, d_a, d_b, d_out, n, stream=None):
        self._check(self._lib.dte_ring_add_device(self._h, _ptr(d_a), _ptr(d_b), _ptr(d_out), int(n),
                                                  _stream(stream)))

    def synth_tuples_device(self, d_tuples, first_tuple, n, num_features, seed, missing_ppm, missing_value, stream=None):
        self._check(self._lib.dte_synth_tuples_device(self._h, _ptr(d_tuples), int(first_tuple), int(n), int(num_features),
                                                      int(seed), int(missing_ppm), int(missing_value),
                                                      _stream(stream)))

    def set_node(self, node_index):
        """Entry of devices_list this engine stands for (0 = host node)."""
        self._check(self._lib.dte_set_node(self._h, int(node_index)))

    def set_kernel_variant(self, variant):
        self._check(self._lib.dte_set_kernel_variant(self._h, int(variant)))

    def autotune(self, n_tuples=0):
        """Time the planner's alternatives on synthetic tuples and pin the fastest; returns the report text."""
        buf = C.create_string_buffer(4096)
        self._check(self._lib.dte_autotune(self._h, int(n_tuples), buf, 4096))
        return buf.value.decode()

    def kernel_name(self):
        return self._name(self._lib.dte_kernel_name)

    def info(self):
        i = DteInfo()
        self._check(self._lib.dte_get_info(self._h, C.byref(i)))
        info = {k: getattr(i, k) for k, _ in DteInfo._fields_}
        info["plan_source"] = PLAN_SOURCES[info["plan_source"]]
        return info
