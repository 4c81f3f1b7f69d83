"""tools/run_sequences.py --check validates a multi-sequence run's inputs without a GPU: frame counts, one image size for
all sequences, distinct names, the calibration and the ground-truth files."""
import os
import struct
import subprocess
import sys
import zlib

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAL = """%YAML:1.0
Camera.fx: 718.856
Camera.fy: 718.856
Camera.cx: 607.1928
Camera.cy: 185.2157
Camera.bf: 386.1448
"""


def _png(path, w, h):
    """A gray 8-bit PNG (colour type 0) written with zlib alone."""
    raw = b"".join(b"\0" + bytes((x * 7 + y * 3) & 255 for x in range(w)) for y in range(h))

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xffffffff)

    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 0, 0, 0, 0)) +
                chunk(b"IDAT", zlib.compress(raw)) + chunk(b"IEND", b""))


def _sequence(root, name, n, w=64, h=40):
    d = os.path.join(root, name)
    for cam in ("image_0", "image_1"):
        os.makedirs(os.path.join(d, cam))
        for k in range(n):
            _png(os.path.join(d, cam, "%06d.png" % k), w, h)
    return d


def _run(*args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_sequences.py"), *args, "--check"],
                       capture_output=True, text=True, cwd=ROOT, timeout=300)
    return r.returncode, r.stdout + r.stderr


def test_check_accepts_sequences_of_unequal_length(built, tmp_path):
    pytest.importorskip("cv2")                       # synth.proj_matrices
    a, b = _sequence(str(tmp_path), "00", 3), _sequence(str(tmp_path), "01", 5)
    cal = tmp_path / "cal.yaml"
    cal.write_text(CAL)
    gt = tmp_path / "gt"
    gt.mkdir()
    for name in ("00", "01"):
        (gt / f"{name}.txt").write_text("1 0 0 0 0 1 0 0 0 0 1 0\n")
    rc, out = _run(a, b, str(cal), "--poses", str(tmp_path / "out"), "--gt", str(gt))
    assert rc == 0, out
    assert "00: 3 stereo pairs of 64x40" in out and "01: 5 stereo pairs of 64x40" in out
    assert not (tmp_path / "out").exists()            # --check writes nothing


def test_check_refuses_bad_inputs(built, tmp_path):
    pytest.importorskip("cv2")
    root = str(tmp_path)
    a = _sequence(root, "00", 3)
    cal = tmp_path / "cal.yaml"
    cal.write_text(CAL)
    out_dir = str(tmp_path / "out")
    rc, out = _run(a, _sequence(root, "01", 3, w=80), str(cal), "--poses", out_dir)
    assert rc != 0 and "one image size" in out
    rc, out = _run(a, _sequence(root, "02", 1), str(cal), "--poses", out_dir)
    assert rc != 0 and "at least two stereo pairs" in out
    os.makedirs(os.path.join(root, "x"))
    rc, out = _run(a, _sequence(os.path.join(root, "x"), "00", 3), str(cal), "--poses", out_dir)
    assert rc != 0 and "collide" in out
    rc, out = _run(a, str(cal), "--poses", out_dir, "--gt", root)
    assert rc != 0 and "no ground truth" in out
    bad = tmp_path / "bad.yaml"
    bad.write_text("Camera.fx: 700\n")
    rc, out = _run(a, str(bad), "--poses", out_dir)
    assert rc != 0 and "missing Camera.fy" in out
