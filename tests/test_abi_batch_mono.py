"""The mono_rotation branch of the batched mode on the CPU: the four entry points are declared, bound with the argument
types of their prototypes and exported; the Python helpers hand the library what the header asks for; and the timing
tool's --check path validates its arguments without a GPU."""
import ctypes as C
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from visual_odom_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "vo_b200.h")).read()
# the prototypes' parameter types, as the header spells them
PROTOS = {
    "vo_batch_mono_rotation": ["vo_ctx*", "int", "int", "const uint8_t*"],
    "vo_batch_wait_mono": ["vo_ctx*", "int", "int", "vo_unit_result*", "vo_mono_result*"],
    "vo_batch_fetch_mono": ["vo_ctx*", "int", "vo_mono_result*", "uint8_t*"],
    "vo_batch_outputs_mono": ["vo_ctx*", "int", "vo_mono_result*", "uint8_t*"],
}
CTYPE = {"vo_ctx*": C.c_void_p, "int": C.c_int, "const uint8_t*": C.c_void_p, "uint8_t*": C.c_void_p,
         "vo_unit_result*": C.POINTER(capi.VoUnitResult), "vo_mono_result*": C.POINTER(capi.VoMonoResult)}


def _params(name):
    m = re.search(r"VO_API int\s+" + name + r"\(([^)]*)\);", HEADER)
    assert m, f"{name} is not declared in include/vo_b200.h"
    return [re.sub(r"\s*\w+$", "", a.strip()).replace(" *", "*") for a in m.group(1).split(",")]


@pytest.mark.parametrize("name", sorted(PROTOS))
def test_declarations_match_the_bindings(name):
    assert _params(name) == PROTOS[name]
    res, args = capi.SIGNATURES[name]
    assert res is C.c_int and len(args) == len(PROTOS[name])
    for got, want in zip(args, PROTOS[name]):
        assert got == CTYPE[want], (name, want, got)


def test_entry_points_are_exported(built):
    lib = C.CDLL(capi.LIB_PATH)
    for name in PROTOS:
        assert hasattr(lib, name), f"{name} is not exported by {capi.LIB_PATH}"


def test_vo_mono_result_layout():
    assert C.sizeof(capi.VoMonoResult) == 4 * 4 + 12 * 8 and capi.VoMonoResult.R.offset == 16


class _Lib:
    """Stands in for the loaded library: records the calls and fills a mono result the way the library would."""

    def __init__(self):
        self.calls = []

    def vo_batch_mono_rotation(self, h, first, n, on):
        self.calls.append(("vo_batch_mono_rotation", first, n, np.ctypeslib.as_array(C.cast(on, C.POINTER(C.c_uint8)), (n,)).copy()))
        return capi.VO_OK

    def vo_batch_wait_mono(self, h, first, n, res, mono):
        self.calls.append(("vo_batch_wait_mono", first, n))
        for i in range(n):
            res[i].n_valid = 10 + i
            mono[i].status, mono[i].n_inliers, mono[i].R[0], mono[i].R[4], mono[i].R[8] = 0, 7 + i, 1.0, 1.0, 1.0
        return capi.VO_OK

    def _fetch(self, name, h, unit, m, mask):
        self.calls.append((name, unit))
        m._obj.n_inliers = 3
        np.ctypeslib.as_array(C.cast(mask, C.POINTER(C.c_uint8)), (8,))[:] = [1, 0, 1, 1, 0, 0, 1, 1]
        return capi.VO_OK

    def vo_batch_fetch_mono(self, *a):
        return self._fetch("vo_batch_fetch_mono", *a)

    def vo_batch_outputs_mono(self, *a):
        return self._fetch("vo_batch_outputs_mono", *a)


def _context():
    c = object.__new__(capi.Context)
    c.h, c.device, c.lib = None, 0, _Lib()
    p = capi.VoParams()
    p.max_features = 64
    c.params = p
    return c


def test_helpers_shapes_and_dtypes():
    c = _context()
    c.batch_mono_rotation(2, [True, 0, 5])
    name, first, n, on = c.lib.calls[-1]
    assert (name, first, n) == ("vo_batch_mono_rotation", 2, 3) and on.tolist() == [1, 0, 1]
    with pytest.raises(ValueError):
        c.batch_mono_rotation(0, [])
    recs, monos = c.batch_wait_mono(4, 2)
    assert len(recs) == len(monos) == 2 and recs[1]["n_valid"] == 11
    m = monos[1]
    assert m["n_inliers"] == 8 and m["R"].shape == (3, 3) and m["R"].dtype == np.float64 and m["t"].shape == (3,)
    assert np.array_equal(m["R"], np.eye(3))
    for fn in (c.batch_fetch_mono, c.batch_outputs_mono):
        f = fn(1, dict(n_valid=5))
        assert f["mono"]["n_inliers"] == 3
        assert f["ess_mask"].dtype == bool and f["ess_mask"].tolist() == [True, False, True, True, False]


TOOL = os.path.join(ROOT, "tools", "batch_mono_timing.py")


def test_timing_tool_check_prints_the_plan():
    out = subprocess.run([sys.executable, TOOL, "--check", "--rounds", "4", "--seconds", "2"], capture_output=True, text=True,
                         timeout=120)
    assert out.returncode == 0, out.stderr
    p = json.loads(out.stdout)["plan"]
    assert p["size"] == [1241, 376] and p["units_per_submission"] == 8 and p["features"] == 2000 and p["in_flight"] == 3
    assert p["rounds"] == 4 and p["seconds"] == 2.0
    assert sorted((m["inputs"], m["units_on"]) for m in p["modes"]) == sorted(
        (i, n) for i in ("host", "device") for n in (0, 1, 8))


@pytest.mark.parametrize("bad", [["--rounds", "2"], ["--seconds", "0"], ["--seconds", "x"]])
def test_timing_tool_check_refuses_bad_arguments(bad):
    out = subprocess.run([sys.executable, TOOL, "--check"] + bad, capture_output=True, text=True, timeout=120)
    assert out.returncode != 0 and "error" in out.stderr
