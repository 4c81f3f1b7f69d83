#!/bin/bash
# demo (needs an H100): writes 8 synthetic KITTI-shaped stereo pairs as PNGs + a calibration file, runs tools/run_sequence.py on them, scores against itself
set -e
D=$(mktemp -d)
python - "$D" <<'PY'
import sys, os, numpy as np, cv2
sys.path.insert(0, os.getcwd())
from visual_odom_b200 import synth
d = sys.argv[1]
os.makedirs(d + "/image_0"); os.makedirs(d + "/image_1")
base = synth.stereo_unit(1241, 376, 31)
frames = [(base["l0"], base["r0"])]
for k in range(1, 8):
    u = synth.stereo_unit(1241, 376, 31, rvec=np.array([0.001, -0.004, 0.0005]) * k, tvec=np.array([0.01, -0.003, -0.2]) * k)
    frames.append((u["l1"], u["r1"]))
for i, (l, r) in enumerate(frames):
    cv2.imwrite(d + "/image_0/%06d.png" % i, l); cv2.imwrite(d + "/image_1/%06d.png" % i, r)
open(d + "/cal.yaml", "w").write("%YAML:1.0\nCamera.fx: 718.8560\nCamera.fy: 718.8560\nCamera.cx: 607.1928\nCamera.cy: 185.2157\nCamera.bf: -386.1448\n")
PY
python tools/run_sequence.py "$D/" "$D/cal.yaml" --poses "$D/out.txt" --threads 4
python tools/run_sequence.py "$D/" "$D/cal.yaml" --gt "$D/out.txt" --threads 4 | tail -2
wc -l "$D/out.txt"
