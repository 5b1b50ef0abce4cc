"""Golden vectors for the dense reward under per-episode coefficients, made by running the REFERENCE'S OWN Python, unmodified.

Runs only in the build container (needs /root/reference); writes tests/golden/dense_options.npz, which travels.  The reference's
FurnitureSawyerDenseRewardEnv runs exactly as in tools/make_golden_dense.py (its Recorder: parent constructor stubbed, the same scripted
world), but every episode draws its own config: the flags at random, every one of the 28 coefficients and thresholds of
config/furniture_sawyer_dense.py:23-70 (ctrl_penalty_coef included) moved off its default.  The coefficients are scaled by a factor in
[1/4, 4] (never 1); the thresholds are drawn in ranges around their defaults wide enough that the script's phase transitions fall
differently: each episode is also run, from the same generator state, with the default coefficients, and the share of episodes whose
phase trace differs is printed and required to be at least half.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from make_golden_dense import OUT, Recorder, draw_flags  # noqa: E402

from furniture_b200.dense import _COEFS, DENSE_DEFAULTS  # noqa: E402

# ranges of the thresholds (defaults: eef_rot 0.95, lift_z 0.02, lift_xy 0.05, align_pos 0.2, align_rot 0.85, move_pos 0.06, move_rot 0.85)
THRESHOLDS = dict(eef_rot_threshold=(0.8, 0.995), lift_z_pos_threshold=(0.005, 0.06), lift_xy_pos_threshold=(0.01, 0.15),
                  align_pos_threshold=(0.05, 0.4), align_rot_threshold=(0.6, 0.98), move_pos_threshold=(0.02, 0.15), move_rot_threshold=(0.6, 0.98))


def draw_config(rng, cfg):
    draw_flags(rng, cfg)
    for k in _COEFS:
        if k in THRESHOLDS:
            v = rng.uniform(*THRESHOLDS[k])
        else:
            f = 1.0
            while abs(np.log(f)) < 0.05:
                f = float(np.exp(rng.uniform(-np.log(4.0), np.log(4.0))))
            v = DENSE_DEFAULTS[k] * f
        assert v != DENSE_DEFAULTS[k]
        setattr(cfg, k, float(v))


def main():
    r = Recorder()
    for k in _COEFS:  # the coefficients the reference reads are the ones this table names, at the defaults of dense.py
        assert float(getattr(r.base_cfg, k)) == DENSE_DEFAULTS[k], k
    rng = np.random.RandomState(20261018)
    coefs, flipped = [], 0
    while len(r.rec["reward"]) < 2000:
        cfg = r.new_config(rng, draw_config)
        twin = type(cfg)(**vars(cfg))
        for k in _COEFS:
            setattr(twin, k, DENSE_DEFAULTS[k])
        state = rng.get_state()
        default_trace = r.episode(rng, twin, record=False)
        rng.set_state(state)
        n0 = len(r.rec["phase"])
        trace = r.episode(rng, cfg)
        flipped += int(trace[n0:] != default_trace)
        coefs.append([getattr(cfg, k) for k in _COEFS])
    share = flipped / r.n_ep
    print("dense_options: %d of %d episodes take other phase transitions than under the default coefficients" % (flipped, r.n_ep))
    assert share >= 0.5, share
    os.makedirs(OUT, exist_ok=True)
    np.savez_compressed(os.path.join(OUT, "dense_options.npz"), **r.arrays(), coef_names=np.array(_COEFS), ep_coefs=np.array(coefs),
                        source="reference furniture/env/furniture_sawyer_dense.py _compute_reward run unmodified on a scripted world, one coefficient "
                               "set per episode (tools/make_golden_dense_options.py)")
    r.report("dense_options")


if __name__ == "__main__":
    main()
