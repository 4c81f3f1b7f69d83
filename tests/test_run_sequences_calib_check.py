"""tools/run_sequences.py --check with --calibration-for NAME=YAML: a per-sequence calibration is accepted and its
matrices printed for that sequence alone, and an unknown dataset name, a missing file or a file without a key are
refused before any GPU work."""
import os
import subprocess
import sys

import pytest

from test_run_sequences_check import CAL, _sequence

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAL04 = CAL.replace("718.856", "707.0912").replace("607.1928", "601.8873").replace("185.2157", "183.1104")


def _run(*args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_sequences.py"), *args, "--check"],
                       capture_output=True, text=True, cwd=ROOT, timeout=300)
    return r.returncode, r.stdout + r.stderr


def test_check_accepts_a_calibration_per_sequence(built, tmp_path):
    pytest.importorskip("cv2")                       # synth.proj_matrices
    a, b = _sequence(str(tmp_path), "00", 3), _sequence(str(tmp_path), "04", 4)
    cal, cal04 = tmp_path / "cal.yaml", tmp_path / "cal04.yaml"
    cal.write_text(CAL)
    cal04.write_text(CAL04)
    rc, out = _run(a, b, str(cal), "--calibration-for", f"04={cal04}", "--poses", str(tmp_path / "out"))
    assert rc == 0, out
    s00, s04 = out.index("00: 3 stereo pairs"), out.index("04: 4 stereo pairs")
    assert f"calibration {cal}" in out[s00:s04] and f"calibration {cal04}" in out[s04:]
    assert "718.856" in out[s00:s04] and "718.856" not in out[s04:] and "707.0912" in out[s04:]
    assert not (tmp_path / "out").exists()            # --check writes nothing


def test_check_refuses_bad_calibration_for(built, tmp_path):
    pytest.importorskip("cv2")
    a, b = _sequence(str(tmp_path), "00", 3), _sequence(str(tmp_path), "04", 3)
    cal = tmp_path / "cal.yaml"
    cal.write_text(CAL)
    out_dir = str(tmp_path / "out")
    rc, out = _run(a, b, str(cal), "--calibration-for", f"05={cal}", "--poses", out_dir)
    assert rc != 0 and "no dataset is named 05" in out
    rc, out = _run(a, b, str(cal), "--calibration-for", f"04={tmp_path / 'none.yaml'}", "--poses", out_dir)
    assert rc != 0 and "does not exist" in out
    bad = tmp_path / "bad.yaml"
    bad.write_text("Camera.fx: 700\n")
    rc, out = _run(a, b, str(cal), "--calibration-for", f"04={bad}", "--poses", out_dir)
    assert rc != 0 and "missing Camera.fy" in out
    rc, out = _run(a, b, str(cal), "--calibration-for", "04", "--poses", out_dir)
    assert rc != 0 and "expected NAME=YAML" in out
