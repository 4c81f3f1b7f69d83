"""tools/run_sequences.py --slots 2 runs four synthetic drives of unequal lengths and two sizes as a queue through two
slots; the pose files are byte for byte those of running all four at once (--mixed-sizes)."""
import os
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest

from visual_odom_b200 import synth
from test_run_sequences_check import CAL

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# (w, h, seed, per-frame rotation, per-frame translation, frames)
DRIVES = [
    (640, 240, 31, (0.001, -0.004, 0.0005), (0.01, -0.003, -0.2), 6),
    (601, 233, 7, (-0.002, 0.003, 0.0), (0.0, 0.0, -0.25), 3),
    (640, 240, 5, (0.002, 0.001, 0.0), (0.0, 0.002, -0.22), 5),
    (601, 233, 23, (-0.001, -0.002, 0.0005), (0.01, 0.0, -0.18), 4),
]


def _png(path, img):
    """A gray 8-bit PNG (colour type 0) written with zlib alone."""
    h, w = img.shape
    raw = b"".join(b"\0" + img[y].tobytes() for y in range(h))

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xffffffff)

    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 0, 0, 0, 0)) +
                chunk(b"IDAT", zlib.compress(raw)) + chunk(b"IEND", b""))


def _drive(root, name, w, h, seed, r, t, n):
    d = os.path.join(root, name)
    for cam in ("image_0", "image_1"):
        os.makedirs(os.path.join(d, cam))
    base = synth.stereo_unit(w, h, seed)
    for k in range(n):
        u = base if k == 0 else synth.stereo_unit(w, h, seed, rvec=np.array(r) * k, tvec=np.array(t) * k)
        left, right = (u["l0"], u["r0"]) if k == 0 else (u["l1"], u["r1"])
        _png(os.path.join(d, "image_0", "%06d.png" % k), left)
        _png(os.path.join(d, "image_1", "%06d.png" % k), right)
    return d


def test_a_queue_through_two_slots_writes_the_poses_of_running_all_at_once(built, tmp_path):
    pytest.importorskip("cv2")                       # synth.proj_matrices
    dirs = [_drive(str(tmp_path), f"{i:02d}", *v) for i, v in enumerate(DRIVES)]
    cal = tmp_path / "cal.yaml"
    cal.write_text(CAL)
    outs = {}
    for mode, extra in (("queue", ["--slots", "2"]), ("all", ["--mixed-sizes"])):
        out = tmp_path / mode
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_sequences.py"), *dirs, str(cal),
                            "--poses", str(out), *extra], capture_output=True, text=True, cwd=ROOT, timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        outs[mode] = out
    for i, v in enumerate(DRIVES):
        a = (outs["queue"] / f"{i:02d}.txt").read_bytes()
        b = (outs["all"] / f"{i:02d}.txt").read_bytes()
        assert a == b, f"drive {i}: pose files differ"
        assert len(a.splitlines()) == v[-1]
    # the poses moved: the drives were tracked, not skipped
    last = np.array((outs["queue"] / "00.txt").read_text().split()[-12:], float).reshape(3, 4)
    assert np.abs(last[:, 3]).max() > 0.1
