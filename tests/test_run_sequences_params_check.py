"""tools/run_sequences.py --check with --params-for NAME=FIELD=V[,...] and --sweep FIELD=V1,V2,...: each sequence's
effective parameters are printed (its own fields over the flags' values), a sweep names one sequence per value after the
first dataset, max_features is raised to the largest bound over the sequences' own bucket grids, and malformed specs,
unknown fields and context-wide fields are refused before any GPU work."""
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


def _params(out, name):
    line = re.search(r"^" + re.escape(name) + r": (fast_threshold=.*)$", out, re.M)
    assert line, out
    return dict(kv.split("=") for kv in line.group(1).split())


@pytest.fixture
def two(tmp_path):
    pytest.importorskip("cv2")                       # synth.proj_matrices
    a, b = _sequence(str(tmp_path), "00", 3), _sequence(str(tmp_path), "04", 4)
    cal = tmp_path / "cal.yaml"
    cal.write_text(CAL)
    return a, b, str(cal), str(tmp_path / "out")


def test_params_for_prints_each_sequences_parameters(built, two):
    a, b, cal, out_dir = two
    rc, out = _run(a, b, cal, "--params-for", "04=fast_threshold=12,lk_epsilon=0.05,features_per_bucket=3",
                   "--refill-threshold", "900", "--poses", out_dir)
    assert rc == 0, out
    p00, p04 = _params(out, "00"), _params(out, "04")
    assert p00["fast_threshold"] == "20" and p00["features_per_bucket"] == "1" and p00["lk_epsilon"] == "0.01"
    assert p04["fast_threshold"] == "12" and p04["features_per_bucket"] == "3" and p04["lk_epsilon"] == "0.05"
    assert p00["refill_threshold"] == p04["refill_threshold"] == "900"      # the flags' value, under its own fields
    assert set(p00) == set(p04) and "lk_win" not in p00 and "max_features" not in p00
    assert "max_features 4096" in out                                      # 187 cells x 3 is below the floor
    assert not os.path.exists(out_dir)


def test_sweep_runs_the_first_dataset_once_per_value_and_raises_max_features(built, two):
    a, b, cal, out_dir = two
    rc, out = _run(a, b, cal, "--sweep", "features_per_bucket=1,8,32", "--poses", out_dir)
    assert rc == 0, out
    for v in ("1", "8", "32"):
        assert _params(out, f"00_features_per_bucket={v}")["features_per_bucket"] == v
    assert "04_" not in out
    # 64 x 40 at rows / 10: (40/4 + 1) x (64/4 + 1) = 187 cells, x 32 per cell
    assert "max_features 5984" in out
    # with --params-for of the first dataset the sweep's field wins, the others stay
    rc, out = _run(a, b, cal, "--params-for", "00=circ_threshold=2,pnp_iterations=700", "--sweep", "pnp_iterations=100,900",
                   "--poses", out_dir)
    assert rc == 0, out
    for v in ("100", "900"):
        p = _params(out, f"00_pnp_iterations={v}")
        assert p["pnp_iterations"] == v and p["circ_threshold"] == "2"


def test_check_refuses_bad_params(built, two):
    a, b, cal, out_dir = two
    cases = [
        (["--params-for", "05=fast_threshold=12"], "no dataset is named 05"),
        (["--params-for", "04=fast_treshold=12"], "no field fast_treshold"),
        (["--params-for", "04=lk_win=15"], "lk_win is context-wide"),
        (["--params-for", "04=max_features=100"], "max_features is context-wide"),
        (["--params-for", "04=fast_nonmax=0"], "fast_nonmax is context-wide"),
        (["--params-for", "04=lk_max_level=2"], "lk_max_level is context-wide"),
        (["--params-for", "04=fast_threshold=abc"], "takes an integer"),
        (["--params-for", "04"], "expected NAME=FIELD=VALUE"),
        (["--params-for", "04=fast_threshold"], "expected FIELD=VALUE"),
        (["--params-for", "04=fast_threshold=12", "--params-for", "04=circ_threshold=1"], "04 is given twice"),
        (["--params-for", "04=bucket_rows_divisor=50"], "too small for the rows/50 bucket size"),
        (["--sweep", "fast_threshold"], "expected FIELD=V1,V2"),
        (["--sweep", "fast_threshold=10,10"], "distinct values"),
        (["--sweep", "lk_win=21,15"], "lk_win is context-wide"),
        (["--sweep", "fast_threshold=10,20", "--slots", "2"], "does not combine with --slots"),
    ]
    for extra, msg in cases:
        rc, out = _run(a, b, cal, *extra, "--poses", out_dir)
        assert rc != 0 and msg in out, (extra, out)
