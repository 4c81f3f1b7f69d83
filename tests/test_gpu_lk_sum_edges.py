"""k_lk_ring at the edges of its choice between the exact integer b sums and cv2's float chains, bit for bit against cv2:
the LK sum-edge fixture (tests/golden/lk_sum_edges/lk_sum_edges.npz, made by tests/golden/make_lk_sum_edges.py) through
vo_lk_track and vo_circular_match under every LK launch configuration, each on a fresh context.  A vote that lets a
rounded chain through, a vote that skips the tail or the b2 chains, or an exact path that combines the chain totals in
another order changes outputs here (tests/test_oracle_lk_sum_edges.py shows it on the oracle)."""
import json
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_lk_sum_edges as ms      # noqa: E402
from test_gpu_lk_edges import CONFIGS, _assert_single       # noqa: E402


@pytest.fixture(scope="module")
def sum_edges(built):
    fx = np.load(ms.OUT)
    out = []
    for ri, r in enumerate(json.loads(str(fx["recipes"]))):
        imgs = ms.mk.images(r)
        assert [ms.mk.sha(a) for a in imgs] == json.loads(str(fx[f"sha256_{ri}"]))
        out.append(dict(imgs=imgs, pts=fx[f"pts_{ri}"], tags=fx[f"tags_{ri}"], out=fx[f"out_{ri}"],
                        status=fx[f"status_{ri}"], err=fx[f"err_{ri}"]))
    return out


def _tags_of(tags, idx):
    return [[t for t in ms.TAGS if tags[i] & ms.BIT[t]] for i in idx[:8]]


@pytest.mark.parametrize("i", range(len(CONFIGS)),
                         ids=["default"] + ["-".join(f"{k}={v}" for k, v in c.items()) for c in CONFIGS[1:]])
def test_sum_edge_fixture_bit_exact(sum_edges, i):
    """The fixture's starts (stored outputs = cv2): call L0 -> R0 through vo_lk_track, the ring through
    vo_circular_match.  A mismatch names the starts and the categories they were mined for."""
    from visual_odom_b200.capi import Context
    c = Context(0, max_features=8192)
    try:
        for k, v in CONFIGS[i].items():
            c.set_option(k, v)
        for ri, e in enumerate(sum_edges):
            imgs, pts, tags = e["imgs"], e["pts"], e["tags"]
            go, gs, ge = c.lk_track(imgs[0], imgs[1], pts)
            bad = np.nonzero((go != e["out"][0]).any(1) | (gs != e["status"][0]))[0]
            assert len(bad) == 0, f"recipe {ri} single call differs at {bad[:8]}, tags {_tags_of(tags, bad)}"
            _assert_single((go, gs, ge), (e["out"][0], e["status"][0], e["err"][0]), f"recipe {ri} single call")
            got = c.circular_match(*imgs, pts)
            for k in range(4):
                bad = np.nonzero((got["raw4"][k] != e["out"][k]).any(1) | (got["status4"][k] != e["status"][k]))[0]
                assert len(bad) == 0, f"recipe {ri}: ring call {k} differs at {bad[:8]}, tags {_tags_of(tags, bad)}"
    finally:
        c.close()
