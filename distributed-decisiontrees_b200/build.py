"""In-tree build of libdte.so for sm_90a (nvcc cross-compiles without a GPU)."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "dte_engine.cu")
DEPS = [SRC, os.path.join(HERE, "csrc", "dte_kernels.cuh"), os.path.join(HERE, "csrc", "dte_device.cuh"),
        os.path.join(HERE, "..", "include", "dte.h"), os.path.join(HERE, "csrc", "dte_partition.hpp"),
        os.path.join(HERE, "csrc", "dte_shap.cuh"), os.path.join(HERE, "csrc", "dte_approx.cuh"),
        os.path.join(HERE, "csrc", "dte_interv.cuh"), os.path.join(HERE, "csrc", "dte_cat.cuh")]
OUT = os.path.join(HERE, "libdte.so")

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    "-std=c++17", "-O3"] + GENCODE + ["-lineinfo",
    "-Xcompiler", "-fPIC", "-shared", "-cudart", "static", "-ldl", "-lpthread",
]


def nvcc_path():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


def stale():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in DEPS)


def build(force=False, verbose=False):
    """Compile csrc/dte_engine.cu -> libdte.so.  Returns the path.  Raises if nvcc is missing."""
    if not force and not stale():
        return OUT
    nvcc = nvcc_path()
    if nvcc is None:
        raise RuntimeError("nvcc not found: cannot build libdte.so (there is no CPU fallback)")
    cmd = [nvcc] + NVCC_FLAGS + ["-o", OUT, SRC]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    env = dict(os.environ)
    # the image exports CC/CXX=/opt/gcc/bin/* wrappers; nvcc should use the system g++
    if os.path.exists("/usr/bin/g++"):
        cmd[1:1] = ["-ccbin", "/usr/bin/g++"]
    res = subprocess.run(cmd, capture_output=True, text=True, env=env)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stderr)
    return OUT


if __name__ == "__main__":
    print(build(force=True, verbose=True))


HOST_SRC = os.path.join(HERE, "..", "tools", "dte_host.cpp")
HOST_OUT = os.path.join(HERE, "..", "tools", "dte_host")


def build_host(force=False):
    """Compile the C++ host program (tools/dte_host.cpp) against libdte.so."""
    if not force and os.path.exists(HOST_OUT) and os.path.getmtime(HOST_OUT) >= max(os.path.getmtime(HOST_SRC), os.path.getmtime(OUT)):
        return HOST_OUT
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    cmd = [gxx, "-O2", "-std=c++17", "-ffp-contract=off", "-o", HOST_OUT, HOST_SRC, "-L" + HERE, "-ldte",
           "-Wl,-rpath," + HERE, "-ldl", "-lpthread", "-lrt"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("g++ failed:\n" + res.stdout + res.stderr)
    return HOST_OUT


MODEL_SRC = os.path.join(HERE, "..", "tools", "dte_model.cpp")
MODEL_OUT = os.path.join(HERE, "..", "tools", "dte_model")


def build_model(force=False):
    """Compile the closed-form performance model CLI (tools/dte_model.cpp; no CUDA needed)."""
    if not force and os.path.exists(MODEL_OUT) and os.path.getmtime(MODEL_OUT) >= os.path.getmtime(MODEL_SRC):
        return MODEL_OUT
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    res = subprocess.run([gxx, "-O2", "-std=c++17", "-o", MODEL_OUT, MODEL_SRC], capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("g++ failed:\n" + res.stdout + res.stderr)
    return MODEL_OUT


def build_host_check(name, force=False):
    """Compile tools/<name>.cu, a host-only checker over the engine headers (runs without a GPU); CPU test tier."""
    src = os.path.join(HERE, "..", "tools", name + ".cu")
    out = os.path.join(HERE, "..", "tools", name)
    deps = [src] + DEPS[1:3] + DEPS[5:]
    if not force and os.path.exists(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps):
        return out
    nvcc = nvcc_path()
    if nvcc is None:
        raise RuntimeError("nvcc not found")
    cmd = [nvcc, "-std=c++17", "-O2"] + GENCODE + ["-cudart", "static", "-o", out, src]
    if os.path.exists("/usr/bin/g++"):
        cmd[1:1] = ["-ccbin", "/usr/bin/g++"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    return out


def build_pack_check(force=False):
    """Host-only checker of the ensemble repacker (tools/pack_check.cu)."""
    return build_host_check("pack_check", force)


def build_plan_check(force=False):
    """Host-only print of the launch planner's decisions (tools/plan_check.cu)."""
    return build_host_check("plan_check", force)


def build_bin_check(force=False):
    """Host-only checker of the binned layout (tools/bin_check.cu)."""
    return build_host_check("bin_check", force)


PART_SRC = os.path.join(HERE, "..", "tools", "partition_check.cpp")
PART_OUT = os.path.join(HERE, "..", "tools", "partition_check")


def build_partition_check(force=False):
    """Brute-force check of csrc/dte_partition.hpp (the data-sharded index arithmetic); CPU test tier."""
    deps = [PART_SRC, os.path.join(HERE, "csrc", "dte_partition.hpp")]
    if not force and os.path.exists(PART_OUT) and all(os.path.getmtime(PART_OUT) >= os.path.getmtime(d) for d in deps):
        return PART_OUT
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    res = subprocess.run([gxx, "-O2", "-std=c++17", "-o", PART_OUT, PART_SRC], capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("g++ failed:\n" + res.stdout + res.stderr)
    return PART_OUT


def build_evidence_tools(force=False):
    """tools/racecheck_canonical (the textbook bulk-copy ring run under racecheck) and tools/pipe_microbench (cycles per
    warp-wide access on the shared-memory / L1 pipe, and the ring fill's L2 -> shared-memory bandwidth with and without
    CTA-cluster multicast): the small CUDA programs behind DESIGN.md §4."""
    nvcc = nvcc_path()
    if nvcc is None:
        raise RuntimeError("nvcc not found")
    outs = []
    for name in ("racecheck_canonical", "pipe_microbench"):
        src = os.path.join(HERE, "..", "tools", name + ".cu")
        out = os.path.join(HERE, "..", "tools", name)
        if force or not os.path.exists(out) or os.path.getmtime(out) < os.path.getmtime(src):
            cmd = [nvcc, "-std=c++17", "-O3"] + GENCODE + ["-lineinfo", "-o", out, src]
            if os.path.exists("/usr/bin/g++"):
                cmd[1:1] = ["-ccbin", "/usr/bin/g++"]
            res = subprocess.run(cmd, capture_output=True, text=True)
            if res.returncode != 0:
                raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
        outs.append(out)
    return outs
