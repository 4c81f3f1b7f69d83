"""The entry points that feed the multi-sequence mode from device memory are exported, declared in the public header and
bound in capi.SIGNATURES with the argument counts of their prototypes, and the torch binding refuses, before any library
call, CPU tensors, a pair count other than the run's sequence count, a pair with one image and an image of another size
than its sequence's."""
import os
import re
import types

import numpy as np
import pytest

from visual_odom_b200 import capi

torch = pytest.importorskip("torch")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMBOLS = {"vo_mseq_begin_device": 9, "vo_mseq_submit_device": 5}


def test_device_entry_points_are_declared_bound_and_exported(built):
    import ctypes as C
    header = open(os.path.join(ROOT, "include", "vo_b200.h")).read()
    lib = C.CDLL(capi.LIB_PATH)
    for name, nargs in SYMBOLS.items():
        m = re.search(r"VO_API int " + name + r"\(([^)]*)\);", header)
        assert m, f"{name} is not declared in include/vo_b200.h"
        assert len(m.group(1).split(",")) == nargs
        assert name in capi.SIGNATURES and len(capi.SIGNATURES[name][1]) == nargs
        assert hasattr(lib, name), f"{name} is not exported by {capi.LIB_PATH}"
    assert "are not accepted in this mode" not in header


class _NoLibrary:
    """Stands in for the loaded library: any entry point reached is a failure of the binding's own checks."""
    def __getattr__(self, name):
        raise AssertionError(f"the binding called {name}")


def _context(sizes, cuda_check=True):
    """A Context with no library and no GPU, in a running multi-sequence run of the given (h, w) sizes.  cuda_check=False
    replaces the CUDA-tensor check by the layout alone, so that CPU tensors reach the size checks."""
    c = object.__new__(capi.Context)
    c.h, c.device, c.lib = None, 0, _NoLibrary()
    c._mseq_n, c._mseq_sizes, c._mseq_keep = len(sizes), list(sizes), [None, None]
    if not cuda_check:
        c._device_image = types.MethodType(lambda self, t, order: capi.image_descriptor(t.shape, t.stride(), 1, order), c)
    return c


def _gray(h, w):
    return torch.zeros(h, w, dtype=torch.uint8)


def test_cpu_tensors_are_refused_before_the_library():
    c = _context([(240, 640)] * 2)
    pairs = [_gray(240, 640), _gray(240, 640)]
    with pytest.raises(TypeError, match="CUDA"):
        c.mseq_submit_device(pairs, pairs)
    with pytest.raises(TypeError, match="CUDA"):
        c.mseq_begin_device(pairs, pairs, np.eye(3, 4), np.eye(3, 4))
    with pytest.raises(TypeError, match="CUDA"):
        c.mseq_submit_device([np.zeros((240, 640), np.uint8)] * 2, [np.zeros((240, 640), np.uint8)] * 2)


def test_pair_counts_and_half_pairs_are_refused_before_the_library():
    c = _context([(240, 640)] * 3, cuda_check=False)
    img = _gray(240, 640)
    with pytest.raises(ValueError, match="for 3 sequences"):
        c.mseq_submit_device([img] * 2, [img] * 2)
    with pytest.raises(ValueError, match="for 3 sequences"):
        c.mseq_submit_device([img] * 4, [img] * 4)
    with pytest.raises(ValueError, match="left and 2 right"):
        c.mseq_submit_device([img] * 3, [img] * 2)
    with pytest.raises(ValueError, match="both images"):
        c.mseq_submit_device([img, None, img], [img, img, img])
    with pytest.raises(ValueError, match="both images"):
        c.mseq_submit_device([img, img, img], [img, img, None])
    with pytest.raises(ValueError, match="both images"):               # a begin takes no retirement
        c.mseq_begin_device([img, None], [img, None], np.eye(3, 4), np.eye(3, 4))
    with pytest.raises(ValueError, match="orders for 3"):
        c.mseq_submit_device([img] * 3, [img] * 3, order=["bgr", "rgb"])
    with pytest.raises(ValueError, match="start needs its first pair"):
        c.mseq_submit_device([img, None, img], [img, None, img], start={1: (np.eye(3, 4), np.eye(3, 4))})


def test_images_of_another_size_are_refused_before_the_library():
    c = _context([(240, 640), (233, 601), None], cuda_check=False)
    a, b = _gray(240, 640), _gray(233, 601)
    with pytest.raises(ValueError, match="sequence 1: image size 640 x 240, the sequence is 601 x 233"):
        c.mseq_submit_device([a, a, None], [a, a, None])
    with pytest.raises(ValueError, match="sequence 0: image size 640 x 241"):
        c.mseq_submit_device([_gray(241, 640), b, None], [_gray(241, 640), b, None])
    with pytest.raises(ValueError, match="sequence 0: image size 601 x 233"):     # a colour layout's size, CHW
        c.mseq_submit_device([torch.zeros(3, 233, 601, dtype=torch.uint8), b, None],
                             [torch.zeros(3, 233, 601, dtype=torch.uint8), b, None], order="rgb")
    with pytest.raises(ValueError, match="left image 640 x 240, right image 601 x 233"):
        c.mseq_submit_device([a, b, None], [b, b, None])
