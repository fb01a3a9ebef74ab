"""Builds tungsten_b200/libtgb200.so (hand-written sm_90a CUDA + host C++) with nvcc, in-tree."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libtgb200.so")
SOURCES = ["tgb200_api.cu", "bvh_build.cpp", "hair_tables.cpp", "sobol_blob.cpp"]
HEADERS = ["tgb_device.cuh", "tgb_wavefront.cuh", "tgb_probe.cuh", "tgb_scene.cuh", "bvh_build.h", "hair_tables.h", os.path.join("..", "..", "include", "tgb200.h")]
BLOB = os.path.join(HERE, "data", "sobol_1024x32.u32")

# -fmad=false: the reference is built without FMA contraction (CMakeLists.txt:17-19); radiance parity needs
# the same rounding.  No --use_fast_math: IEEE division / sqrt.
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-fmad=false",
              "--prec-div=true", "--prec-sqrt=true", "-Xcompiler", "-fPIC,-O3,-ffp-contract=off",
              "-Xptxas", "-v", "--shared", '-DTGB_SOBOL_BLOB_PATH="%s"' % BLOB]


# Variants that build() makes next to the library, for tests that load them with TGB200_LIB.  smem4: four traversal stack
# entries per lane in shared memory instead of 32, so every walk deeper than four nodes runs through the local-memory half of
# TravStack (tests/test_gpu_tree_shapes.py requires its answers to equal the library's byte for byte).
CHECKED_VARIANTS = {"smem4": ["TGB_SMEM_STACK=4"]}


def variant_path(name):
    return os.path.join(HERE, "libtgb200_%s.so" % name)


def needs_build(out=OUT):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [BLOB, os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def _nvcc(out, defines=()):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + ["-D" + d for d in defines] + [os.path.join(CSRC, s) for s in SOURCES] + ["-o", out, "-ccbin", "/usr/bin/g++"]
    return cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)


def build_variant(name, defines):
    """Experimental build with extra -D flags -> tungsten_b200/libtgb200_<name>.so (load with TGB200_LIB)."""
    out = variant_path(name)
    _, p = _nvcc(out, defines)
    text = p.communicate()[0]
    if p.returncode != 0:
        sys.stderr.write(text)
        raise RuntimeError("nvcc failed")
    return out


def build(force=False, verbose=False):
    """The library and CHECKED_VARIANTS, compiled side by side (each is one long single-threaded ptxas run)."""
    jobs = []
    if force or needs_build():
        jobs.append((OUT, os.path.join(HERE, "build.log")) + _nvcc(OUT))
    for name, defines in CHECKED_VARIANTS.items():
        if force or needs_build(variant_path(name)):
            jobs.append((variant_path(name), os.path.join(HERE, "build_%s.log" % name)) + _nvcc(variant_path(name), defines))
    failed = []
    for out, log, cmd, p in jobs:
        text = p.communicate()[0]
        with open(log, "w") as f:
            f.write(" ".join(cmd) + "\n" + text)
        if verbose or p.returncode != 0:
            sys.stderr.write(text)
        if p.returncode != 0:
            failed.append(log)
    if failed:
        raise RuntimeError("nvcc failed, see %s" % ", ".join(failed))
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
