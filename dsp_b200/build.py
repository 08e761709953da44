"""Build libdspb200.so (hand-written CUDA, sm_90a only) in-tree with nvcc.

`python -m dsp_b200.build` or `from dsp_b200.build import build; build()`.
The .so is a build product (git-ignored): every checkout builds its own.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SOURCES = ["api.cu", "fir.cu", "biquad.cu", "resample.cu", "design.cu", "delay.cu", "edge.cu"]
OUT = os.path.join(HERE, "libdspb200.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _newest(paths):
    return max(os.path.getmtime(p) for p in paths)


def build_variant(name, defines):
    """A measurement variant of the library (compile-time knobs), dsp_b200/variants/libdspb200_<name>.so; select it
    at run time with DSP_B200_LIB=<path>."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    vdir = os.path.join(HERE, "variants")
    os.makedirs(vdir, exist_ok=True)
    out = os.path.join(vdir, "libdspb200_%s.so" % name)
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    cmd = [nvcc, "-shared", "-Xcompiler", "-fPIC", "-O3", "-std=c++17", "-lineinfo"] + ARCH + ["-D" + d for d in defines] + srcs + ["-o", out]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("nvcc failed building variant " + name)
    return out


def build(force=False, verbose=False):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    srcs = [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    deps = srcs + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    deps.append(os.path.join(HERE, "..", "include", "dsp_b200.h"))
    deps.append(os.path.abspath(__file__))   # ARCH and the flags: a library built with other ones is stale
    if not force and os.path.exists(OUT) and os.path.getmtime(OUT) >= _newest(deps):
        return OUT
    if not os.path.exists(nvcc):
        if os.path.exists(OUT):
            return OUT  # GPU box without a toolkit: use the prebuilt library that travelled
        raise RuntimeError("nvcc not found and no prebuilt libdspb200.so")
    cmd = [nvcc, "-shared", "-Xcompiler", "-fPIC", "-O3", "-std=c++17", "-lineinfo"] + ARCH
    if verbose:
        cmd += ["-Xptxas", "-v"]
    cmd += srcs + ["-o", OUT]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if verbose or r.returncode != 0:
        sys.stderr.write(r.stdout)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed building libdspb200.so")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
