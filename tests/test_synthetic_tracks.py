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
