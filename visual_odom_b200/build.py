"""Build the in-tree native artefacts.

  visual_odom_b200/csrc/*.cu   -> visual_odom_b200/libvo_b200.so   (nvcc, sm_90a only)
  oracle/*.c                   -> oracle/_build/liboracle.so       (gcc; test infrastructure)

Both are plain compiler invocations (no cmake, no JIT cache) so the built .so files travel to the
GPU box with the repo snapshot.  `python -m visual_odom_b200.build` rebuilds what is stale: an artefact is rebuilt
when the contents of its inputs or its command differ from those recorded when it was built (a SHA-256 stamp under
csrc/_obj/stamps/), never because of file times alone.
"""
import hashlib
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


def _rel(s):
    return s.replace(REPO + os.sep, "")


def _digest(inputs, cmd):
    h = hashlib.sha256("\0".join(_rel(c) for c in cmd).encode())
    for p in inputs:
        h.update(_rel(p).encode() + b"\0")
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def _stamp(target):
    return os.path.join(OBJ, "stamps", _rel(target).replace(os.sep, "__") + ".sha256")


def _stale(inputs, target, cmd):
    """True if `target` is missing or was built from other input contents or by another command.  File times are not
    consulted: copying a built tree, checking files out again or restoring them changes times, not what a build makes,
    and must not send a rebuild into a tree the caller may be unable to write."""
    if not os.path.exists(target):
        return True
    try:
        with open(_stamp(target)) as f:
            return f.read() != _digest(inputs, cmd)
    except OSError:
        return True


def _record(inputs, target, cmd):
    os.makedirs(os.path.dirname(_stamp(target)), exist_ok=True)
    with open(_stamp(target), "w") as f:
        f.write(_digest(inputs, cmd))


def _build(inputs, target, cmd, what, force=False):
    """Run `cmd` (which writes `target`) unless `target` is up to date with `inputs`; True if it ran."""
    if not (force or _stale(inputs, target, cmd)):
        return False
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError(what)
    _record(inputs, target, cmd)
    return True


def build_native(verbose=False, force=False):
    srcs = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))
    hdrs = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh")))
    hdrs.append(os.path.join(REPO, "include", "vo_b200.h"))
    hdrs.append(os.path.abspath(__file__))          # the flags above
    os.makedirs(OBJ, exist_ok=True)
    jobs = []
    for s in srcs:
        o = os.path.join(OBJ, os.path.basename(s)[:-3] + ".o")
        cmd = [NVCC] + NVCC_FLAGS + ["-c", s, "-o", o]
        if force or _stale([s] + hdrs, o, cmd):
            jobs.append(([s] + hdrs, o, cmd))

    def run(job):
        inputs, o, cmd = job
        full = cmd[:1] + (["-Xptxas", "-v"] if verbose else []) + cmd[1:]
        return job, full, subprocess.run(full, capture_output=True, text=True)

    with ThreadPoolExecutor(max_workers=8) as ex:
        for (inputs, o, cmd), full, r in ex.map(run, jobs):
            if verbose or r.returncode != 0:
                sys.stderr.write(" ".join(full) + "\n" + r.stdout + r.stderr)
            if r.returncode != 0:
                raise RuntimeError("nvcc failed: " + " ".join(full))
            _record(inputs, o, cmd)
    objs = [os.path.join(OBJ, os.path.basename(s)[:-3] + ".o") for s in srcs]
    cmd = [NVCC, "-shared"] + GENCODE + ["-cudart", "static", "-o", LIB] + objs + ["-lz", "-lpthread"]
    _build(objs, LIB, cmd, "link failed", force)
    return LIB


FACADE_LIB = os.path.join(ROOT, "libvo_facade.so")
FACADE_TEST = os.path.join(REPO, "tests", "cpp", "facade_main")
UTILS_TEST = os.path.join(REPO, "tests", "cpp", "utils_main")


def build_facade(force=False):
    """The reference-signature C++ facade (include/compat/*.h) over libvo_b200.so + its test driver."""
    src = os.path.join(CSRC, "facade.cpp")
    inc = os.path.join(REPO, "include", "compat")
    deps = [src, LIB] + sorted(os.path.join(inc, f) for f in os.listdir(inc))
    cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I", inc, src, "-o", FACADE_LIB,
           "-L", ROOT, "-lvo_b200", "-Wl,-rpath,$ORIGIN"]
    _build(deps, FACADE_LIB, cmd, "facade build failed", force)
    for main, exe, what in (("facade_main.cpp", FACADE_TEST, "facade test driver build failed"),
                            ("utils_main.cpp", UTILS_TEST, "utils test driver build failed")):
        tsrc = os.path.join(REPO, "tests", "cpp", main)
        cmd = ["g++", "-O2", "-std=c++17", "-I", inc, tsrc, "-o", exe, "-L", ROOT, "-lvo_facade", "-lvo_b200",
               "-Wl,-rpath,$ORIGIN/../../visual_odom_b200"]
        _build([tsrc, FACADE_LIB], exe, cmd, what, force)
    return FACADE_LIB


def build_hostcheck(force=False):
    """pnp_math.cuh (and the other *_math.cuh) compiled for the host (g++), used by the CPU tests to check the kernels' math."""
    src = os.path.join(CSRC, "host_check.cpp")
    dep = [src] + [os.path.join(CSRC, f) for f in ("pnp_math.cuh", "ess_math.cuh", "p3p_math.cuh", "remap_math.cuh")]
    cmd = ["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", src, "-o", HOSTCHECK_LIB]
    _build(dep, HOSTCHECK_LIB, cmd, "hostcheck build failed", force)
    return HOSTCHECK_LIB


def build_oracle(force=False):
    srcs = sorted(os.path.join(ORACLE_DIR, f) for f in os.listdir(ORACLE_DIR) if f.endswith(".c"))
    os.makedirs(os.path.dirname(ORACLE_LIB), exist_ok=True)
    # -ffp-contract=off: the restatement must round like the (FMA-less) reference build
    cmd = ["gcc", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-o", ORACLE_LIB] + srcs + ["-lm"]
    _build(srcs, ORACLE_LIB, cmd, "oracle build failed", force)
    return ORACLE_LIB


if __name__ == "__main__":
    v = "-v" in sys.argv
    f = "-f" in sys.argv
    print(build_native(verbose=v, force=f))
    print(build_hostcheck(force=f))
    print(build_facade(force=f))
    print(build_oracle(force=f))
