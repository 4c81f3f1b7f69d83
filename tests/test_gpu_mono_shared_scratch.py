"""The sequence modes and the batched mode run trackingFrame2Frame's mono_rotation branch in the same per-unit scratch
blocks.  On one context: a batched submission with some units switched on, a vo_seq_* mono sequence, a vo_mseq_* mono
run with more buffer units than the batch (so the blocks grow), and the batched submission again.  Every step gives what
it gives on a fresh context, bit for bit (records, mono results, essential masks, point lists), at the same
kernel_launches() delta."""
import numpy as np
import pytest

from visual_odom_b200 import synth

pytestmark = pytest.mark.gpu

W, H = 640, 240
B = 4                                   # batched units: the vo_mseq_* run below takes 2 * 3 = 6 buffer units
ON = [1, 0, 1, 1]
N_SEL = 300
T_PREV = (0.0, 0.0, -0.8)
FRAMES = 4
# (seed, per-frame rotation, per-frame translation)
DRIVES = [
    (31, (0.001, -0.004, 0.0005), (0.01, -0.003, -0.2)),
    (7, (-0.002, 0.003, 0.0), (0.0, 0.0, -0.25)),
    (13, (0.0, 0.002, -0.001), (-0.02, 0.004, -0.15)),
]


def _drive(seed, r, t):
    out = [None] * FRAMES
    for k in range(FRAMES):
        u = synth.stereo_unit(W, H, seed, rvec=np.array(r) * k, tvec=np.array(t) * k)
        out[k] = (u["l0"], u["r0"]) if k == 0 else (u["l1"], u["r1"])
    return out


@pytest.fixture(scope="module")
def data():
    base = synth.stereo_unit(W, H, 0)
    units = [dict(synth.stereo_unit(W, H, 500 + i), n_select=N_SEL, t_prev=T_PREV) for i in range(B)]
    return dict(P_l=base["P_l"], P_r=base["P_r"], units=units, drives=[_drive(*d) for d in DRIVES])


def _context():
    from visual_odom_b200.capi import Context
    return Context(0, max_features=2048)


def _configure(c, d):
    c.batch_configure(W, H, B, d["P_l"], d["P_r"])
    c.batch_mono_rotation(0, ON)
    return c.make_units(d["units"])


def _batch(c, d, units):
    """A submission of the B units: records, mono results, masks and lists."""
    arr, keep, pitch = units
    c.batch_submit(arr, 0, pitch)
    recs, monos = c.batch_wait_mono(0, B)
    out = []
    for u in range(B):
        f = c.batch_fetch_mono(u, recs[u])
        out.append(dict(rec=recs[u], mono=monos[u], fetched=f["mono"], ess_mask=f["ess_mask"], lists=c.batch_fetch(u, recs[u])))
    return out


def _seq(c, d):
    """vo_seq_* with the option "mono_rotation" on drive 0: per frame the record (mono result and mask included)."""
    fr = d["drives"][0]
    c.set_option("mono_rotation", 1)
    try:
        c.seq_begin(fr[0][0], fr[0][1], d["P_l"], d["P_r"])
        return [c.seq_push(*fr[k], mono=True) for k in range(1, FRAMES)]
    finally:
        c.set_option("mono_rotation", 0)


def _mseq(c, d):
    """vo_mseq_* with the flag VO_MSEQ_MONO_ROTATION on every drive: per frame the records."""
    frs = d["drives"]
    c.mseq_begin([f[0][0] for f in frs], [f[0][1] for f in frs], d["P_l"], d["P_r"], mono_rotation=True)
    out = []
    for k in range(1, FRAMES):
        c.mseq_submit([f[k][0] for f in frs], [f[k][1] for f in frs])
        out.append(c.mseq_wait(mono=True))
    return out


def _same(a, b, where):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), where
        for k in a:
            _same(a[k], b[k], f"{where}: {k}")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, f"{where}[{i}]")
    else:
        x, y = np.asarray(a), np.asarray(b)
        assert x.dtype == y.dtype and np.array_equal(x, y), where


def _launches(c, step):
    l0 = c.kernel_launches()
    out = step()
    return out, c.kernel_launches() - l0


def test_the_modes_share_the_scratch_blocks_bit_for_bit(built, data):
    from visual_odom_b200 import capi
    fresh = {}
    for name, step in (("batch", _batch), ("seq", _seq), ("mseq", _mseq)):
        f = _context()
        try:
            args = (_configure(f, data),) if name == "batch" else ()
            fresh[name] = _launches(f, lambda: step(f, data, *args))
        finally:
            f.close()
    c = _context()
    try:
        units = _configure(c, data)
        # the second batched submission reads the switch table set before the sequences ran
        for name, step, args in (("batch", _batch, (units,)), ("seq", _seq, ()), ("mseq", _mseq, ()), ("batch", _batch, (units,))):
            got, n = _launches(c, lambda: step(c, data, *args))
            want, n_fresh = fresh[name]
            _same(got, want, name)
            assert n == n_fresh > 0, (name, n, n_fresh)
    finally:
        c.close()
    # the branch ran: units switched off report zeros, and the others and the sequences found essential matrices
    batch = fresh["batch"][0]
    assert all(not batch[u]["mono"]["status"] and not batch[u]["mono"]["R"].any() for u in range(B) if not ON[u])
    assert any(batch[u]["mono"]["status"] == capi.VO_OK and batch[u]["mono"]["n_inliers"] > 0 for u in range(B) if ON[u])
    seq = fresh["seq"][0] + [r for recs in fresh["mseq"][0] for r in recs]
    assert any(r["mono"]["status"] == capi.VO_OK and r["mono"]["n_inliers"] > 0 for r in seq)
