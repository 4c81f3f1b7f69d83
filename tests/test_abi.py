"""The C-ABI library loads on a CPU-only host and exports every symbol include/vo_b200.h declares.
No compute call is made here (there is no CPU fallback to call)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    txt = open(os.path.join(ROOT, "include", "vo_b200.h")).read()
    return sorted(set(re.findall(r"VO_API\s+[\w\s\*]+?\b(vo_\w+)\s*\(", txt)))


def test_header_symbols_are_exported(built):
    from visual_odom_b200 import capi
    lib = ctypes.CDLL(capi.LIB_PATH)
    names = declared_symbols()
    assert len(names) >= 19
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/vo_b200.h but not exported"
        assert n in capi.SIGNATURES, f"{n} missing from the ctypes signature table"


def test_library_does_not_link_libcuda(built):
    """cuTensorMapEncodeTiled is resolved at run time so the .so loads where no driver is installed."""
    import subprocess
    from visual_odom_b200 import capi
    out = subprocess.run(["ldd", capi.LIB_PATH], capture_output=True, text=True).stdout
    assert "libcuda.so" not in out and "libcudart" not in out


def test_default_params_match_reference_literals(built):
    from visual_odom_b200 import capi
    lib = capi.load_library()
    p = capi.VoParams()
    lib.vo_default_params(ctypes.byref(p))
    assert (p.fast_threshold, p.fast_nonmax, p.lk_win, p.lk_max_level, p.lk_max_iters) == (20, 1, 21, 3, 30)
    assert (p.lk_epsilon, p.lk_min_eig, p.circ_threshold, p.pnp_iterations) == (0.01, 0.001, 0, 500)
    assert p.pnp_reproj_error == 0.5
    import numpy as np
    assert p.pnp_confidence == float(np.float32(0.999))      # `float confidence = 0.999;` visualOdometry.cpp:170


def test_no_gpu_fails_loudly(built):
    """Without a CUDA device vo_create must fail with a message -- never fall back to the CPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from visual_odom_b200.capi import Context, VoError
    with pytest.raises(VoError) as e:
        Context(0)
    assert "no CPU fallback" in str(e.value) or "CUDA" in str(e.value)


def test_sass_has_tma_and_no_legacy_tensor_ops(built):
    """The LK kernel stages windows with TMA (UTMALDG); nothing here uses tensor cores."""
    import shutil
    import subprocess
    if not shutil.which("cuobjdump"):
        pytest.skip("cuobjdump not available")
    from visual_odom_b200 import capi
    sass = subprocess.run(["cuobjdump", "-sass", capi.LIB_PATH], capture_output=True, text=True).stdout
    assert "UTMALDG" in sass
    elfs = subprocess.run(["cuobjdump", "-lelf", capi.LIB_PATH], capture_output=True, text=True).stdout.splitlines()
    assert elfs and all(ln.endswith(".sm_90a.cubin") for ln in elfs), elfs


def test_result_record_numpy_view_matches_the_ctypes_struct():
    """capi.RESULT_DTYPE (what batch_wait / dist_gather_wait hand out with raw=True) is the C record, field for field."""
    import ctypes as C
    import numpy as np
    from visual_odom_b200 import capi
    res = (capi.VoUnitResult * 3)()
    for i, r in enumerate(res):
        r.n_features, r.n_detected, r.n_tracked, r.n_valid, r.n_inliers, r.ransac_iters, r.pnp_status = [10 * i + k for k in range(7)]
        for k in range(3):
            r.rvec[k] = 0.5 * i + k; r.tvec[k] = -1.0 * i - k
        for k in range(9):
            r.R[k] = 100 * i + k
    arr = np.frombuffer(res, dtype=capi.RESULT_DTYPE)
    assert arr.dtype.itemsize == C.sizeof(capi.VoUnitResult) == 152
    a = capi.Context.records_to_dicts(arr)
    b = [capi.Context._result_dict(r) for r in res]
    for x, y in zip(a, b):
        assert set(x) == set(y)
        for k in x:
            assert np.array_equal(x[k], y[k]), k
        assert x["R"].shape == (3, 3) and isinstance(x["n_valid"], int)
