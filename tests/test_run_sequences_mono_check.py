"""tools/run_sequences.py --check --mono-rotation validates the inputs without a GPU and reports the rotation source."""
import os
import subprocess
import sys

from test_run_sequences_check import CAL, ROOT, _sequence


def test_check_accepts_mono_rotation(tmp_path):
    a = _sequence(str(tmp_path), "00", 3)
    b = _sequence(str(tmp_path), "01", 2)
    cal = tmp_path / "cal.yaml"
    cal.write_text(CAL)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_sequences.py"), a, b, str(cal),
                        "--poses", str(tmp_path / "out"), "--check", "--mono-rotation"], capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr
    assert "00: 3 stereo pairs of 64x40" in r.stdout and "01: 2 stereo pairs" in r.stdout
    assert "recoverPose (mono_rotation = true)" in r.stdout
    assert not (tmp_path / "out").exists()
