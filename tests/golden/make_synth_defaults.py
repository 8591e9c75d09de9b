"""Write synth_defaults.npz: the output of synth_bal / synth_config with default options on a few seeds and shapes.

tests/test_synthetic_tracks.py::test_default_output_is_byte_identical compares the generator against it bit for bit, so an
option added to synth_bal cannot change the problems that the existing tests and bench.py draw."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

CASES = {
    "tiny": dict(nc=12, nl=60, mean_n=4.1, seed=1),
    "small": dict(nc=49, nl=120, mean_n=4.1, seed=38401),
    "tracks": dict(nc=14, nl=9, mean_n=0.0, seed=1008, track_lengths=[8] * 9, lm_spread=0.5),
    "wide": dict(nc=20, nl=80, mean_n=6.0, seed=5, max_tan=1.5, normalize_scale=None),
}
CONFIGS = {"ladybug": ("ladybug-49", 0.05), "trafalgar": ("trafalgar-257", 0.01)}
FIELDS = ("cams", "lms", "lm_off", "obs_cam", "obs_xy")


def compute():
    from rootba_b200.synthetic import synth_bal, synth_config
    out = {}
    for name, kw in CASES.items():
        kw = dict(kw)
        a = synth_bal(kw.pop("nc"), kw.pop("nl"), kw.pop("mean_n"), **kw)
        out.update({f"{name}/{f}": getattr(a, f) for f in FIELDS})
    for name, (cfg, scale) in CONFIGS.items():
        a = synth_config(cfg, scale=scale)
        out.update({f"{name}/{f}": getattr(a, f) for f in FIELDS})
    return out


if __name__ == "__main__":
    np.savez_compressed(os.path.join(HERE, "synth_defaults.npz"), **compute())
