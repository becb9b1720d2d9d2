"""Builds rnnoise_b200/librnnoise_b200.so in-tree: host C (gcc) + CUDA for sm_90a (nvcc).

  nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo --fmad=false ...
--fmad=false is part of the arithmetic contract (DESIGN.md "Numerics"): the reference's DSP code is
compiled without FMA contraction; every FMA the kernels execute is an explicit fmaf().
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "librnnoise_b200.so")
# Tolerance-build experiment (VERDICT r1 item 4): the same sources with FMA contraction allowed in the DSP code.
# NOT the product: it breaks the bit-exact contract (DESIGN.md "Numerics"); tools/tolerance_experiment.py loads it
# through $RNNOISE_B200_LIB_PATH to measure what the contract costs and what contraction does to pitch parity.
SO_FMAD = os.path.join(HERE, "librnnoise_b200_fmad.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _newer(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def sources():
    out = []
    for d in (CSRC, os.path.join(HERE, "..", "include")):
        for f in sorted(os.listdir(d)):
            if f.endswith((".c", ".cu", ".cuh", ".h", ".hpp")):
                out.append(os.path.join(d, f))
    return out


def build(force=False, verbose=False, fmad=False, variant=None, flags=()):
    """variant / flags: an experimental build librnnoise_b200_<variant>.so with extra nvcc flags (compile-time knobs
    such as -DPG=8), loaded through $RNNOISE_B200_LIB_PATH by the A/B tools; never the product library."""
    so = SO_FMAD if fmad else os.path.join(HERE, f"librnnoise_b200_{variant}.so") if variant else SO
    if not force and not _newer(so, sources() + [os.path.abspath(__file__)]):
        return so
    obj = os.path.join(HERE, "build_fmad" if fmad else f"build_{variant}" if variant else "build")
    os.makedirs(obj, exist_ok=True)
    cmds = []
    cobjs = []
    for c in ("rnnoise_api.c", "model_blob.c"):
        o = os.path.join(obj, c + ".o")
        cmds.append(["gcc", "-O2", "-fPIC", "-pthread", "-Wall", "-fvisibility=hidden", "-DRNNOISE_BUILD", "-c", os.path.join(CSRC, c), "-o", o])
        cobjs.append(o)
    eo = os.path.join(obj, "engine.cu.o")
    extra = os.environ.get("RNNOISE_B200_NVCC_FLAGS", "").split() + list(flags)
    cmds.append([NVCC, *ARCH, *extra, "-O3", "-lineinfo", "--fmad=true" if fmad else "--fmad=false", "-Xcompiler", "-fPIC,-fvisibility=hidden", "-DRNNOISE_BUILD",
                 "-Xptxas", "-v" if verbose else "-O3", "-c", os.path.join(CSRC, "engine.cu"), "-o", eo])
    cmds.append([NVCC, *ARCH, "-shared", "-o", so, *cobjs, eo, "-cudart", "static", "-lpthread"])
    for cmd in cmds:
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or r.returncode:
            sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        if r.returncode:
            raise RuntimeError("build of librnnoise_b200.so failed")
    return so


if __name__ == "__main__":
    var = sys.argv[sys.argv.index("--variant") + 1] if "--variant" in sys.argv else None
    fl = sys.argv[sys.argv.index("--flags") + 1].split() if "--flags" in sys.argv else []
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, fmad="--fmad" in sys.argv, variant=var, flags=fl))
