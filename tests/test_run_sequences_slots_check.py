"""tools/run_sequences.py --slots N --check: the datasets form a queue, each starting in the first slot that frees (the
lowest slot on a tie) at the submission after its predecessor's last frame; the schedule is printed without a GPU, more
datasets than one context's sequence limit are accepted, and N outside 1..64 is refused."""
import os
import re
import subprocess
import sys

import pytest

from test_run_sequences_check import CAL, _sequence

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(*args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "run_sequences.py"), *args, "--check"],
                       capture_output=True, text=True, cwd=ROOT, timeout=300)
    return r.returncode, r.stdout + r.stderr


def _schedule(out):
    return {m[0]: (int(m[1]), int(m[2]), int(m[3])) for m in re.findall(r"^  (\S+): slot (\d+), submissions (\d+)\.\.(\d+)$", out, re.M)}


def test_slots_check_prints_the_queue_schedule(built, tmp_path):
    pytest.importorskip("cv2")                       # synth.proj_matrices
    lengths = [5, 2, 3, 4, 2]
    dirs = [_sequence(str(tmp_path), f"{i:02d}", n, w=64 + 8 * (i % 2)) for i, n in enumerate(lengths)]
    cal = tmp_path / "cal.yaml"
    cal.write_text(CAL)
    rc, out = _run(*dirs, str(cal), "--slots", "2", "--poses", str(tmp_path / "out"))
    assert rc == 0, out
    # 00 (5 frames) slot 0 at 1..5; 01 (2) slot 1 at 1..2; 02 (3) slot 1 at 3..5; 03 (4): both free at 6 -> slot 0
    # at 6..9; 04 (2) slot 1 at 6..7
    assert _schedule(out) == {"00": (0, 1, 5), "01": (1, 1, 2), "02": (1, 3, 5), "03": (0, 6, 9), "04": (1, 6, 7)}, out
    assert "schedule: 5 sequences through 2 slots of 72x40, 9 submissions" in out
    assert not (tmp_path / "out").exists()            # --check writes nothing
    rc, out = _run(*dirs, str(cal), "--slots", "5", "--poses", str(tmp_path / "out"))
    assert rc == 0 and all(v[0] == i and v[1] == 1 for i, v in enumerate(_schedule(out).values())), out


def test_slots_accept_more_datasets_than_one_run_holds(built, tmp_path):
    pytest.importorskip("cv2")
    dirs = [_sequence(str(tmp_path), f"{i:02d}", 2) for i in range(66)]
    cal = tmp_path / "cal.yaml"
    cal.write_text(CAL)
    rc, out = _run(*dirs, str(cal), "--slots", "64", "--poses", str(tmp_path / "out"))
    assert rc == 0, out
    s = _schedule(out)
    assert s["64"] == (0, 3, 4) and s["65"] == (1, 3, 4)
    rc, out = _run(*dirs, str(cal), "--poses", str(tmp_path / "out"))
    assert rc != 0 and "at most 64" in out, out


@pytest.mark.parametrize("n", ["0", "65", "-1"])
def test_slots_outside_one_to_64_are_refused(built, tmp_path, n):
    pytest.importorskip("cv2")
    a = _sequence(str(tmp_path), "00", 3)
    cal = tmp_path / "cal.yaml"
    cal.write_text(CAL)
    rc, out = _run(a, str(cal), "--slots", n, "--poses", str(tmp_path / "out"))
    assert rc != 0 and f"--slots {n}" in out and "1 to 64" in out, out
