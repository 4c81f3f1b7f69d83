"""tools/run_sequences.py --mixed-sizes --check: sequences of different image sizes are accepted and every size is
printed; sizes with different pyramid depths are refused; without the flag the one-size refusal names it."""
import os
import subprocess
import sys

import pytest

from test_run_sequences_check import CAL, _sequence

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(*args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_sequences.py"), *args, "--check"],
                       capture_output=True, text=True, cwd=ROOT, timeout=300)
    return r.returncode, r.stdout + r.stderr


def test_mixed_sizes_check_accepts_and_prints_every_size(built, tmp_path):
    pytest.importorskip("cv2")                       # synth.proj_matrices
    a, b = _sequence(str(tmp_path), "00", 3), _sequence(str(tmp_path), "01", 4, w=80)
    cal = tmp_path / "cal.yaml"
    cal.write_text(CAL)
    rc, out = _run(a, b, str(cal), "--mixed-sizes", "--poses", str(tmp_path / "out"))
    assert rc == 0, out
    assert "00: 3 stereo pairs of 64x40" in out and "01: 4 stereo pairs of 80x40" in out
    assert "image sizes: 00 64x40, 01 80x40" in out
    assert not (tmp_path / "out").exists()            # --check writes nothing


def test_mixed_sizes_check_refuses_mixed_pyramid_depths(built, tmp_path):
    pytest.importorskip("cv2")
    a, b = _sequence(str(tmp_path), "00", 3), _sequence(str(tmp_path), "01", 3, w=120, h=60)   # 1 and 2 levels
    cal = tmp_path / "cal.yaml"
    cal.write_text(CAL)
    rc, out = _run(a, b, str(cal), "--mixed-sizes", "--poses", str(tmp_path / "out"))
    assert rc != 0 and "pyramid" in out and "120x60" in out and "64x40" in out, out


def test_without_the_flag_the_refusal_names_it(built, tmp_path):
    pytest.importorskip("cv2")
    a, b = _sequence(str(tmp_path), "00", 3), _sequence(str(tmp_path), "01", 3, w=80)
    cal = tmp_path / "cal.yaml"
    cal.write_text(CAL)
    rc, out = _run(a, b, str(cal), "--poses", str(tmp_path / "out"))
    assert rc != 0 and "one image size" in out and "--mixed-sizes" in out, out
