"""synth_bal with chosen track lengths: the lengths survive generation exactly, observations stay valid, bad input raises."""
import numpy as np
import pytest

from rootba_b200.synthetic import project, synth_bal


@pytest.mark.parametrize("n,count,nc", [(2, 33, 12), (17, 3, 30), (65, 2, 71), (300, 2, 306)])
def test_track_lengths_are_exact(n, count, nc):
    want = np.full(count, n)
    want[-1] = 2  # a mixed list keeps its order
    a = synth_bal(nc, count, 0.0, seed=n, track_lengths=want, lm_spread=0.5)
    assert a.nl == count and np.array_equal(a.track_lengths(), want)
    lm_of_obs = np.repeat(np.arange(a.nl), want)
    for l in range(a.nl):  # distinct cameras, ascending, in range
        c = a.obs_cam[a.lm_off[l]:a.lm_off[l + 1]]
        assert np.all(np.diff(c) > 0) and c[0] >= 0 and c[-1] < nc
    # after normalisation and perturbation every landmark is still in front of every observing camera
    _, z = project(a.cams[a.obs_cam], a.lms[lm_of_obs])
    assert np.all(z > 0)


def test_default_draw_is_unchanged():
    """without track_lengths the generator consumes the same random stream as before (the fixtures stay the same)"""
    a = synth_bal(49, 300, 4.1, seed=7)
    b = synth_bal(49, 300, 4.1, seed=7, lm_spread=3.0)
    assert np.array_equal(a.lm_off, b.lm_off) and np.array_equal(a.obs_xy, b.obs_xy)
    assert a.track_lengths().min() >= 2 and len(np.unique(a.track_lengths())) > 3


def test_rejects_bad_track_lengths():
    with pytest.raises(ValueError):
        synth_bal(10, 3, 0.0, track_lengths=[2, 3])        # one entry per landmark
    with pytest.raises(ValueError):
        synth_bal(10, 2, 0.0, track_lengths=[1, 3])        # n >= 2
    with pytest.raises(ValueError):
        synth_bal(10, 2, 0.0, track_lengths=[11, 3])       # n <= nc
    with pytest.raises(ValueError):                        # a wide spread pushes observations out of the field of view
        synth_bal(40, 200, 0.0, seed=1, track_lengths=np.full(200, 30), lm_spread=30.0)


def test_default_output_is_byte_identical():
    """the options added to synth_bal (k1_sigma, k2_sigma, tracks) leave every problem drawn with their defaults bit for bit as
    it was (tests/golden/synth_defaults.npz, written by tests/golden/make_synth_defaults.py before they existed)"""
    import importlib.util
    import os
    from conftest import ROOT
    spec = importlib.util.spec_from_file_location("mk", os.path.join(ROOT, "tests", "golden", "make_synth_defaults.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    got = mk.compute()
    ref = np.load(os.path.join(ROOT, "tests", "golden", "synth_defaults.npz"))
    assert sorted(got) == sorted(ref.files)
    for k in ref.files:
        assert got[k].dtype == ref[k].dtype and np.array_equal(got[k], ref[k]), k


def test_chosen_tracks_distortion_and_turned_cameras():
    from rootba_b200.synthetic import turn_cameras_around
    tracks = [[0, 3, 5], [1, 2], [5, 4, 0, 2], [3, 4]]
    a = synth_bal(6, 4, 0.0, seed=3, tracks=tracks, lm_spread=0.5, k1_sigma=0.2, k2_sigma=0.05)
    for l, t in enumerate(tracks):
        assert np.array_equal(a.obs_cam[a.lm_off[l]:a.lm_off[l + 1]], sorted(t))
    assert np.abs(a.cams[:, 8]).max() > 0.05 and np.abs(a.cams[:, 9]).max() > 0.01
    b = turn_cameras_around(a, [0, 4])
    lm_of_obs = np.repeat(np.arange(a.nl), a.track_lengths())
    _, za = project(a.cams[a.obs_cam], a.lms[lm_of_obs])
    xyb, zb = project(b.cams[b.obs_cam], b.lms[lm_of_obs])
    turned = np.isin(a.obs_cam, [0, 4])
    assert np.all(za > 0) and np.all(zb[turned] < 0) and np.allclose(zb, np.where(turned, -za, za))
    assert np.array_equal(b.cams[:, 7:], a.cams[:, 7:]) and np.array_equal(b.obs_xy, a.obs_xy)
    assert np.array_equal(b.cams[[1, 2, 3, 5]], a.cams[[1, 2, 3, 5]])
    # the turned camera centres stay where they were
    from rootba_b200.synthetic import quat_to_rot
    ca = -np.einsum("mji,mj->mi", quat_to_rot(a.cams[:, :4]), a.cams[:, 4:7])
    cb = -np.einsum("mji,mj->mi", quat_to_rot(b.cams[:, :4]), b.cams[:, 4:7])
    assert np.allclose(ca, cb, rtol=1e-12, atol=1e-9)
    with pytest.raises(ValueError):
        synth_bal(6, 1, 0.0, tracks=[[0, 6]])
