"""Build the in-tree native artefacts.

  visual_odom_b200/csrc/*.cu   -> visual_odom_b200/libvo_b200.so   (nvcc, sm_90a only)
  oracle/*.c                   -> oracle/_build/liboracle.so       (gcc; test infrastructure)

Both are plain compiler invocations (no cmake, no JIT cache) so the built .so files travel to the
GPU box with the repo snapshot.  `python -m visual_odom_b200.build` rebuilds what is stale.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(ROOT)
CSRC = os.path.join(ROOT, "csrc")
OBJ = os.path.join(CSRC, "_obj")
LIB = os.path.join(ROOT, "libvo_b200.so")
HOSTCHECK_LIB = os.path.join(ROOT, "libvo_hostcheck.so")
ORACLE_DIR = os.path.join(REPO, "oracle")
ORACLE_LIB = os.path.join(ORACLE_DIR, "_build", "liboracle.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]    # H100 only; no PTX for other archs
NVCC_FLAGS = GENCODE + [
    "-lineinfo", "-O3", "-std=c++17",
    "-fmad=false",            # IEEE mul/add kept separate: parity with the CPU reference needs it
    "-Xcompiler", "-fPIC,-fvisibility=hidden",
    "-cudart", "static",
]


def _newer(src_list, target):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in src_list)


def build_native(verbose=False, force=False):
    srcs = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    hdrs.append(os.path.join(REPO, "include", "vo_b200.h"))
    hdrs.append(os.path.abspath(__file__))          # the flags above
    os.makedirs(OBJ, exist_ok=True)
    jobs = []
    for s in srcs:
        o = os.path.join(OBJ, os.path.basename(s)[:-3] + ".o")
        if force or _newer([s] + hdrs, o):
            cmd = [NVCC] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + \
                ["-c", s, "-o", o]
            jobs.append(cmd)

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        return cmd, r

    with ThreadPoolExecutor(max_workers=8) as ex:
        for cmd, r in ex.map(run, jobs):
            if verbose or r.returncode != 0:
                sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
            if r.returncode != 0:
                raise RuntimeError("nvcc failed: " + " ".join(cmd))
    objs = [os.path.join(OBJ, os.path.basename(s)[:-3] + ".o") for s in srcs]
    if force or jobs or _newer(objs, LIB):
        cmd = [NVCC, "-shared"] + GENCODE + ["-cudart", "static",
               "-o", LIB] + objs + ["-lz", "-lpthread"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return LIB


FACADE_LIB = os.path.join(ROOT, "libvo_facade.so")
FACADE_TEST = os.path.join(REPO, "tests", "cpp", "facade_main")
UTILS_TEST = os.path.join(REPO, "tests", "cpp", "utils_main")


def build_facade(force=False):
    """The reference-signature C++ facade (include/compat/*.h) over libvo_b200.so + its test driver."""
    src = os.path.join(CSRC, "facade.cpp")
    inc = os.path.join(REPO, "include", "compat")
    deps = [src, LIB] + [os.path.join(inc, f) for f in os.listdir(inc)]
    if force or _newer(deps, FACADE_LIB):
        cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I", inc, src, "-o", FACADE_LIB,
               "-L", ROOT, "-lvo_b200", "-Wl,-rpath,$ORIGIN"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("facade build failed")
    tsrc = os.path.join(REPO, "tests", "cpp", "facade_main.cpp")
    if force or _newer([tsrc, FACADE_LIB], FACADE_TEST):
        cmd = ["g++", "-O2", "-std=c++17", "-I", inc, tsrc, "-o", FACADE_TEST, "-L", ROOT, "-lvo_facade", "-lvo_b200",
               "-Wl,-rpath,$ORIGIN/../../visual_odom_b200"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("facade test driver build failed")
    usrc = os.path.join(REPO, "tests", "cpp", "utils_main.cpp")
    if force or _newer([usrc, FACADE_LIB], UTILS_TEST):
        cmd = ["g++", "-O2", "-std=c++17", "-I", inc, usrc, "-o", UTILS_TEST, "-L", ROOT, "-lvo_facade", "-lvo_b200",
               "-Wl,-rpath,$ORIGIN/../../visual_odom_b200"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("utils test driver build failed")
    return FACADE_LIB


def build_hostcheck(force=False):
    """pnp_math.cuh compiled for the host (g++), used by the CPU tests to check the kernels' math."""
    src = os.path.join(CSRC, "host_check.cpp")
    dep = [src] + [os.path.join(CSRC, f) for f in ("pnp_math.cuh", "ess_math.cuh", "p3p_math.cuh")]
    if force or _newer(dep, HOSTCHECK_LIB):
        cmd = ["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", src,
               "-o", HOSTCHECK_LIB]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("hostcheck build failed")
    return HOSTCHECK_LIB


def build_oracle(force=False):
    srcs = sorted(os.path.join(ORACLE_DIR, f) for f in os.listdir(ORACLE_DIR) if f.endswith(".c"))
    os.makedirs(os.path.dirname(ORACLE_LIB), exist_ok=True)
    if force or _newer(srcs, ORACLE_LIB):
        # -ffp-contract=off: the restatement must round like the (FMA-less) reference build
        cmd = ["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", ORACLE_LIB] + srcs + ["-lm"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("oracle build failed")
    return ORACLE_LIB


if __name__ == "__main__":
    v = "-v" in sys.argv
    f = "-f" in sys.argv
    print(build_native(verbose=v, force=f))
    print(build_hostcheck(force=f))
    print(build_facade(force=f))
    print(build_oracle(force=f))
