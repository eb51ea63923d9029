"""CPU: pin the oracle (oracle/s2o_solver.c) to the unmodified reference (oracle/_ref) bit for bit at step settings other
than (1/60 s, 4 sub-steps, 2 relax iterations, warm starting on), for every solver variant.

Much of a step depends on these settings: the hertz clamps of the soft variants (contact and joint hertz against a fraction
of the sub-step rate), the shape of each variant's program (no relax sweep at E = 0, TGS_Soft's relax-store fold with a
segment run S - 1 times), and the body damping 1 / (1 + h * damping) with h = dt / S. SETTINGS is chosen so that every
hertz clamp is reached on both sides (contact hertz 30, joint hertz 60, reference src/core.h):

    (1/60, 1, 0, on)   TGS_Soft contact clamp (0.25 * 60 = 15 Hz); SoftStep contact and joint clamps; no relax sweep
    (1/60, 1, 1, on)   TGS_Soft folds its store into the last relax sweep behind a segment run S - 1 = 0 times
    (1/30, 2, 3, on)   a coarse step with a long relax
    (1/60, 3, 0, off)  no relax sweep (the bias sweep writes the warm-start impulses); cold start; SoftStep joints at 45 Hz
    (1/60, 8, 1, on)   TGS_Soft joint clamp on its boundary (0.125 * 480 = 60 Hz); the sub-step count of BASELINE config 2
    (1/120, 8, 2, on)  TGS_Soft joints at their constant 60 Hz; PGS_Soft / Jacobi contacts constant, joints on the boundary
    (1/240, 4, 5, on)  a fine step with many relax sweeps; PGS_Soft / Jacobi joints at their constant 60 Hz

scenes.damped_mix gives every body damping and a gravity scale (the pyramid and the chains have neither), so a wrong h in
the damping or a swapped coefficient changes the result."""
import pytest

from solver2d_b200 import scenes
from test_oracle_cpu import VARIANTS, _pin

# (dt, sub-steps, relax iterations, warm starting)
SETTINGS = [(1.0 / 60.0, 1, 0, True), (1.0 / 60.0, 1, 1, True), (1.0 / 30.0, 2, 3, True), (1.0 / 60.0, 3, 0, False),
            (1.0 / 60.0, 8, 1, True), (1.0 / 120.0, 8, 2, True), (1.0 / 240.0, 4, 5, True)]
SETTING_IDS = ["dt60-S1-E0", "dt60-S1-E1", "dt30-S2-E3", "dt60-S3-E0-cold", "dt60-S8-E1", "dt120-S8-E2", "dt240-S4-E5"]


def _damped_joints(lib, solver):
    return scenes.damped_mix(lib, solver, joints=True)


SCENES = {
    "pyramid": (scenes.pyramid, dict(base_count=10), 40),
    "limited_chains": (scenes.limited_chains, {}, 40),
    "damped_mix": (scenes.damped_mix, {}, 40),
    "damped_mix_joints": (_damped_joints, {}, 40),
}


@pytest.mark.parametrize("setting", SETTINGS, ids=SETTING_IDS)
@pytest.mark.parametrize("scene", sorted(SCENES))
@pytest.mark.parametrize("solver", VARIANTS)
def test_oracle_pinned_at_step_settings(reference, solver, scene, setting):
    """Reference steps at the setting (warm starting on), then one stage solved by the oracle and the reference at the
    setting: bodies and manifold impulses bit for bit."""
    recipe, kw, warm = SCENES[scene]
    dt, S, E, warm_start = setting
    # the reference's Jacobi variant blows piles apart within a few steps (its own behaviour): pin it early
    nc, nj = _pin(reference, recipe, solver, 2 if solver == "Jacobi" else warm, S, E, warm_start=warm_start, dt=dt, **kw)
    assert nc > 0
    assert nj == {"pyramid": 0, "limited_chains": 19, "damped_mix": 0, "damped_mix_joints": 6}[scene]



@pytest.mark.parametrize("solver", VARIANTS)
def test_oracle_pinned_paused(reference, solver):
    """A paused step (dt = 0): the reference still runs the solver, with inv_dt = 0 and h = 0 (XPBD leaves early)."""
    nc, _ = _pin(reference, scenes.damped_mix, solver, 2 if solver == "Jacobi" else 40, 4, 2, dt=0.0)
    assert nc > 0
