"""Tracking parameters per slot / unit (vo_mseq_params, vo_batch_params): both entry points are declared, bound with the
argument counts of their prototypes and exported; the structs they sit beside keep their layout (vo_params and
vo_mseq_start against the header, field for field); and the Python helpers fill every field a caller does not name from
the context's own vo_params before any library call."""
import ctypes as C
import os
import re

import pytest

from visual_odom_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = open(os.path.join(ROOT, "include", "vo_b200.h")).read()
SYMBOLS = {"vo_mseq_params": 4, "vo_batch_params": 4}
CTYPES = {"int": C.c_int, "float": C.c_float, "double": C.c_double}


def test_entry_points_are_declared_bound_and_exported(built):
    lib = C.CDLL(capi.LIB_PATH)
    for name, nargs in SYMBOLS.items():
        m = re.search(r"VO_API int\s+" + name + r"\(([^)]*)\);", HEADER)
        assert m, f"{name} is not declared in include/vo_b200.h"
        args = [a.strip() for a in m.group(1).split(",")]
        assert len(args) == nargs and args[-1] == "const vo_params* p", args
        assert name in capi.SIGNATURES and len(capi.SIGNATURES[name][1]) == nargs
        assert capi.SIGNATURES[name][1][3]._type_ is capi.VoParams
        assert hasattr(lib, name), f"{name} is not exported by {capi.LIB_PATH}"


def _struct_fields(name):
    body = re.search(r"typedef struct " + name + r" \{(.*?)\} " + name + ";", HEADER, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for ctype, names in re.findall(r"^\s*(int|float|double)\s+([^;]+);", body, re.M):
        for d in names.split(","):
            m = re.fullmatch(r"\s*(\w+)(?:\[(\d+)\])?\s*", d)
            fields.append((ctype, m.group(1), m.group(2)))
    return fields


def test_vo_params_layout_is_the_headers():
    fields = _struct_fields("vo_params")
    assert [f[1] for f in fields] == [f[0] for f in capi.VoParams._fields_]
    for (ctype, name, _), (_, ct) in zip(fields, capi.VoParams._fields_):
        assert CTYPES[ctype] is ct, name
    # unchanged: the four bookkeeping fields stay the last ones, after max_units
    assert capi.VoParams.max_units.offset == 68 and capi.VoParams.bucket_age_threshold.offset == 84
    assert C.sizeof(capi.VoParams) == 88


def test_vo_mseq_start_layout_is_the_headers():
    fields = _struct_fields("vo_mseq_start")
    assert [f[1] for f in fields] == [f[0] for f in capi.VoMseqStart._fields_] == ["slot", "w", "h", "P_l", "P_r"]
    assert [int(f[2] or 1) for f in fields] == [1, 1, 1, 12, 12]
    assert capi.VoMseqStart.P_l.offset == 12 and capi.VoMseqStart.P_r.offset == 60 and C.sizeof(capi.VoMseqStart) == 108


class _Recorder:
    """Stands in for the loaded library: records the vo_params arrays the binding passes."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(h, first, n, arr):
            self.calls.append((name, first, n, [arr[i] for i in range(n)]))
            return capi.VO_OK
        return call


def _context(**prm):
    c = object.__new__(capi.Context)
    c.h, c.device, c.lib = None, 0, _Recorder()
    p = capi.VoParams()
    for k, v in dict(dict(fast_threshold=20, fast_nonmax=1, lk_win=21, lk_max_level=3, lk_max_iters=30, lk_epsilon=0.01,
                          lk_min_eig=0.001, circ_threshold=0, pnp_iterations=500, pnp_reproj_error=0.5,
                          pnp_confidence=0.999, max_features=8192, max_units=1, refill_threshold=2000,
                          bucket_rows_divisor=10, features_per_bucket=1, bucket_age_threshold=10), **prm).items():
        setattr(p, k, v)
    c.params = p
    return c


def _as_dict(p):
    return {f: getattr(p, f) for f, _ in capi.VoParams._fields_}


@pytest.mark.parametrize("method,entry", [("mseq_params", "vo_mseq_params"), ("batch_params", "vo_batch_params")])
def test_helpers_fill_unnamed_fields_from_the_contexts_params(method, entry):
    c = _context(max_features=4096, pnp_iterations=300, lk_max_level=2)
    getattr(c, method)(5, [dict(fast_threshold=12, features_per_bucket=3), None, {}])
    (name, first, n, got), = c.lib.calls
    assert (name, first, n) == (entry, 5, 3)
    own = _as_dict(c.params)
    assert _as_dict(got[0]) == dict(own, fast_threshold=12, features_per_bucket=3)
    assert _as_dict(got[1]) == own and _as_dict(got[2]) == own
    assert own["max_features"] == 4096 and own["lk_max_level"] == 2       # the context's, not the library defaults
    # the context's own params are left alone
    assert c.params.fast_threshold == 20 and c.params.features_per_bucket == 1


@pytest.mark.parametrize("method", ["mseq_params", "batch_params"])
def test_helpers_refuse_unknown_fields_and_empty_lists(method):
    c = _context()
    with pytest.raises(TypeError, match="fast_treshold"):
        getattr(c, method)(0, [dict(fast_treshold=12)])
    with pytest.raises(ValueError):
        getattr(c, method)(0, [])
    assert c.lib.calls == []
