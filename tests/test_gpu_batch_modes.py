"""The whole path through the benchmark's own entry points (vo_frame_batch, vo_batch_submit / vo_batch_wait /
vo_batch_outputs) under every scheduling option, against the reference path (cv2 through oracle/ref_path.py).

Every configuration gets a fresh context.  Units are KITTI-size with 2000 features and ranges hold 4 of them, so a range
has 8000 features: more than the resident LK warps under any SM partition, so its launch splits feature-rings into
work items.  For every unit the record and the point lists of vo_batch_fetch must match the oracle (indices, the four
lists, points3D and inliers bit-exact, [R|t] within 1e-4), and the packed lists of vo_batch_outputs must equal
vo_batch_fetch.  Consecutive configurations put different units into the same slots, so a launch that skipped work
cannot pass on what an earlier context left in recycled device memory.

The packed-output block is sized by the largest feature bound of the resident slots; the mixed-count tests submit
ranges of 2000 and 300 features in the orders that once retired a pending submission, dropped waited lists or packed a
re-run at the smaller count.
"""
import numpy as np
import pytest

from test_gpu_path import check_unit, reference_unit          # the whole-path oracle and its comparison, shared
from test_gpu_seq import _frames as sequence_frames
from visual_odom_b200 import synth

pytestmark = pytest.mark.gpu

W, H, B = 1241, 376, 4
N_SEL, N_SMALL = 2000, 300
T_PREV = (0.0, 0.0, -0.8)
OUT_BYTES_PER_SLOT = 4 * 8 + 4 + 12 + 4        # float2 pts4[4] | int kept_idx | float3 X | int inlier (batch.cu)
LISTS = ("l0", "r0", "l1", "r1", "kept_idx", "X", "inliers")


@pytest.fixture(scope="module")
def pool(built):
    """Three sets of B units at N_SEL features and two at N_SMALL, with the reference path of each, computed once."""
    pytest.importorskip("cv2")

    def make(seed0, n_sets, n_sel):
        sets = []
        for k in range(n_sets):
            us = [synth.stereo_unit(W, H, seed0 + B * k + i, cal=synth.KITTI00) for i in range(B)]
            sets.append(dict(units=us, n_sel=n_sel, refs=[reference_unit(u, n_sel, np.array(T_PREV)) for u in us]))
        return sets
    return dict(big=make(60, 3, N_SEL), small=make(90, 2, N_SMALL))


def _context(**opts):
    from visual_odom_b200.capi import Context
    c = Context(0, max_features=2048)
    for k, v in opts.items():
        c.set_option(k, v)
    return c


def _arr(c, s):
    return c.make_units([dict(u, n_select=s["n_sel"], t_prev=T_PREV) for u in s["units"]])


def _submit(c, s, slot0):
    arr, keep, pitch = _arr(c, s)
    c.batch_submit(arr, slot0, pitch)
    return keep


def _check(c, slot0, res, s, outputs=True, per=None):
    """Records + vo_batch_fetch of the units in slots [slot0, slot0 + B) against the oracle of set `s`, and
    vo_batch_outputs against vo_batch_fetch.  `per`: the packed point slots a unit must take in the D2H copy."""
    for i, (r, ref) in enumerate(zip(res, s["refs"])):
        got = c.batch_fetch(slot0 + i, r)
        check_unit(r, got, ref)
        if outputs:
            o = c.batch_outputs(slot0 + i, r)
            for k in LISTS:
                assert np.array_equal(o[k], got[k]), (slot0 + i, k)
            if per is not None:
                assert o["d2h_bytes"] == (per * OUT_BYTES_PER_SLOT + 255) // 256 * 256


@pytest.mark.parametrize("streams", [1, 2])
def test_frame_batch(pool, streams):
    big = pool["big"]
    c = _context(batch_streams=streams)
    try:
        c.batch_configure(W, H, 2 * B, big[0]["units"][0]["P_l"], big[0]["units"][0]["P_r"])
        for a, b in ((streams % 3, (streams + 1) % 3), ((streams + 2) % 3, streams % 3)):     # two calls, other units in the slots
            s = dict(units=big[a]["units"] + big[b]["units"], n_sel=N_SEL, refs=big[a]["refs"] + big[b]["refs"])
            arr, keep, pitch = _arr(c, s)
            res = c.frame_batch(arr, pitch)
            for i, (r, ref) in enumerate(zip(res, s["refs"])):
                check_unit(r, c.batch_fetch(i, r), ref)
    finally:
        c.close()


SUBMIT_CONFIGS = {
    "partition-auto": {},
    "partition+8": {"sm_partition": 8},
    "partition-off": {"sm_partition": 0},      # the high-priority helper streams
    "graphs-0": {"graphs": 0},
}


@pytest.mark.parametrize("name", list(SUBMIT_CONFIGS))
def test_two_submissions_in_flight(pool, name):
    """Two ranges submitted before either is waited for, twice, with other units in the slots the second time (a
    captured graph is then replayed on new data)."""
    big = pool["big"]
    k = list(SUBMIT_CONFIGS).index(name)
    c = _context(batch_outputs=1, **SUBMIT_CONFIGS[name])
    try:
        c.batch_configure(W, H, 2 * B, big[0]["units"][0]["P_l"], big[0]["units"][0]["P_r"])
        for step in range(2):
            sa, sb = big[(k + 2 * step) % 3], big[(k + 2 * step + 1) % 3]
            keep = [_submit(c, sa, 0), _submit(c, sb, B)]
            _check(c, 0, c.batch_wait(0, B), sa, per=2048)
            _check(c, B, c.batch_wait(B, B), sb, per=2048)
            del keep
    finally:
        c.close()


def test_three_submissions_in_flight_and_resident_rerun(pool):
    """The benchmark's e2e loop: three ranges in flight, then a re-run of what is resident (units = NULL) submitted
    while the other two are still in flight.  A negative SM count for the partition is refused and changes nothing."""
    from visual_odom_b200.capi import VO_E_INVALID, VoError
    big = pool["big"]
    c = _context(batch_outputs=1)
    try:
        with pytest.raises(VoError) as e:
            c.set_option("sm_partition", -8)
        assert e.value.code == VO_E_INVALID
        c.batch_configure(W, H, 3 * B, big[0]["units"][0]["P_l"], big[0]["units"][0]["P_r"])
        keep = [_submit(c, big[(j + 1) % 3], j * B) for j in range(3)]
        _check(c, 0, c.batch_wait(0, B), big[1], per=2048)
        c.batch_submit(None, 0, 0, n_units=B)
        _check(c, B, c.batch_wait(B, B), big[2], per=2048)
        _check(c, 2 * B, c.batch_wait(2 * B, B), big[0], per=2048)
        _check(c, 0, c.batch_wait(0, B), big[1], per=2048)
        del keep
    finally:
        c.close()


# ---- packed outputs of ranges with different feature counts ---------------------------------------------------------
def test_pending_submissions_survive_other_feature_counts(pool):
    """A submission of another feature count while one is in flight: the one in flight stays pending and its lists
    stay valid, whether the packed block has to grow (300 then 2000) or keeps its size (2000 then 300)."""
    big, small = pool["big"], pool["small"]
    c = _context(batch_outputs=1)
    try:
        c.batch_configure(W, H, 2 * B, big[0]["units"][0]["P_l"], big[0]["units"][0]["P_r"])
        keep = [_submit(c, small[0], 0), _submit(c, big[0], B)]
        _check(c, 0, c.batch_wait(0, B), small[0])
        _check(c, B, c.batch_wait(B, B), big[0], per=2048)
        keep = [_submit(c, big[1], 0), _submit(c, small[1], B)]
        _check(c, 0, c.batch_wait(0, B), big[1], per=2048)
        _check(c, B, c.batch_wait(B, B), small[1])
        del keep
    finally:
        c.close()


def test_waited_lists_survive_a_smaller_submission(pool):
    """A waited unit stays readable until its own slots are resubmitted, whatever is submitted to other slots."""
    big, small = pool["big"], pool["small"]
    c = _context(batch_outputs=1)
    try:
        c.batch_configure(W, H, 2 * B, big[0]["units"][0]["P_l"], big[0]["units"][0]["P_r"])
        keep = [_submit(c, big[2], 0)]
        res_a = c.batch_wait(0, B)
        keep.append(_submit(c, small[0], B))
        _check(c, 0, res_a, big[2], per=2048)
        _check(c, B, c.batch_wait(B, B), small[0], per=2048)
        del keep
    finally:
        c.close()


def test_resident_rerun_after_a_smaller_submission(pool):
    """Re-running a resident range (units = NULL) after a smaller submission to other slots tracks and packs it at its
    own feature count."""
    big, small = pool["big"], pool["small"]
    c = _context(batch_outputs=1)
    try:
        c.batch_configure(W, H, 2 * B, big[0]["units"][0]["P_l"], big[0]["units"][0]["P_r"])
        keep = [_submit(c, big[1], 0)]
        _check(c, 0, c.batch_wait(0, B), big[1], per=2048)
        keep.append(_submit(c, small[1], B))
        _check(c, B, c.batch_wait(B, B), small[1])
        c.batch_submit(None, 0, 0, n_units=B)
        _check(c, 0, c.batch_wait(0, B), big[1], per=2048)
        del keep
    finally:
        c.close()


# ---- sequence mode -----------------------------------------------------------------------------------------------------
def test_sequence_without_graphs_equals_graph_path(built):
    """vo_seq_push with plain launches (graphs = 0) gives the records, point lists, pose and carried state of the
    graph path.  Both contexts stay open, so neither runs on memory the other left behind."""
    from visual_odom_b200.capi import Context
    base, frames = sequence_frames(W, H, 7, 9)
    ctxs = [Context(0, max_features=8192), Context(0, max_features=8192)]
    try:
        ctxs[1].set_option("graphs", 0)
        runs = []
        for c in ctxs:
            c.seq_begin(frames[0][0], frames[0][1], base["P_l"], base["P_r"])
            runs.append(([c.seq_push(l, r) for l, r in frames[1:]], c.seq_pose(), c.seq_state()))
        (ref, pose_ref, state_ref), (got, pose, state) = runs
        for k, (a, b) in enumerate(zip(got, ref)):
            for key in ("n_features", "n_detected", "n_tracked", "n_valid", "n_inliers", "ransac_iters"):
                assert a[key] == b[key], (k, key)
            for key in ("l0", "r0", "l1", "r1", "R", "tvec", "rvec"):
                assert np.array_equal(a[key], b[key]), (k, key)
        assert all(r["n_valid"] > 50 for r in ref)
        assert np.array_equal(pose, pose_ref)
        assert all(np.array_equal(a, b) for a, b in zip(state, state_ref))
    finally:
        for c in ctxs:
            c.close()
